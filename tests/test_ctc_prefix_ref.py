"""CPU checks of CTC prefix scoring as tests/ctc_prefix_ref.py restates it (DESIGN.md 4.9) -- the definition the CUDA kernels
(csrc/ctc_prefix.cu) are tested against in tests/test_gpu_ctc_prefix.py: brute-force enumeration, the prefix invariant and
nn.functional.ctc_loss at real sizes, -inf handling, the joint beam step at weight 0, and the recognizer's argument checks."""
import itertools
import math
from types import SimpleNamespace

import pytest
import torch

from oracle.beam_search import beam_step
from tests import ctc_prefix_ref as cpr

EOS = cpr.EOS


def _lp(T, V, seed, scale=2.0):
    g = torch.Generator().manual_seed(seed)
    return torch.log_softmax(scale * torch.randn(T, V, generator=g, dtype=torch.float64), dim=-1)


@pytest.mark.parametrize('T,V,seed', [(6, 3, 0), (5, 4, 1), (3, 4, 2), (1, 4, 3)])
def test_psi_equals_the_enumerated_prefix_probability(T, V, seed):
    """Every V ** T path, collapsed: psi of every prefix of up to 3 labels (repeats included) is the probability that the
    labels start with it, and psi of a prefix completed by <S/E> is the probability that they equal it."""
    lp = _lp(T, V, seed)
    paths = cpr.enumerate_labels(lp)
    assert abs(sum(paths.values()) - 1.0) < 1e-12
    for L in (1, 2, 3):
        for h in itertools.product(range(1, V), repeat=L):
            want = sum(p for labels, p in paths.items() if labels[:L] == h)
            _, psi = cpr.prefix_state(lp, T, list(h), eos=None)
            assert abs(math.exp(float(psi)) - want) < 1e-10, (h, float(psi), want)
            if h[-1] == EOS:
                _, psi_end = cpr.prefix_state(lp, T, list(h))
                assert abs(math.exp(float(psi_end)) - paths.get(h, 0.0)) < 1e-10, h


def test_prefix_invariant_and_ctc_loss_at_real_sizes():
    """exp psi(g) = P(labels == g) + sum over c of exp psi(g c), every c as a prefix; psi(g <S/E>) = -ctc_loss of g <S/E>."""
    T, V = 50, 40
    g = torch.Generator().manual_seed(5)
    lens = [50, 37, 21, 9]
    for b, Tb in enumerate(lens):
        lp = _lp(T, V, 10 + b)
        toks = torch.randint(2, V, (6,), generator=g).tolist()
        toks[3] = toks[2]                                          # a repeated token
        for L in (0, 1, 4, 6):
            gamma, psi = cpr.prefix_state(lp, Tb, toks[:L], eos=None)
            _, ext = cpr.extend(lp, Tb, gamma, L == 0, toks[L - 1] if L else -1, list(range(1, V)), eos=None)
            rhs = torch.logsumexp(torch.cat((cpr.total(gamma).view(1), ext)), dim=0)
            assert abs(float(psi) - float(rhs)) < 1e-9, (b, L, float(psi), float(rhs))
            if L == 0:                                             # every label sequence starts with the empty prefix
                assert float(psi) == 0.0
            _, psi_end = cpr.prefix_state(lp, Tb, toks[:L] + [EOS])
            nll = torch.nn.functional.ctc_loss(lp[:, None, :], torch.tensor([toks[:L] + [EOS]]), torch.tensor([Tb]),
                                               torch.tensor([L + 1]), blank=0, reduction='sum', zero_infinity=False)
            assert abs(float(psi_end) + float(nll)) < 1e-9 * max(1.0, abs(float(nll))), (b, L)


def test_impossible_prefixes_are_minus_infinity_never_nan():
    lp = _lp(6, 5, 7)
    # more labels than frames
    gamma, psi = cpr.prefix_state(lp, 2, [2, 3, 4], eos=None)
    assert float(psi) == float('-inf') and not bool(torch.isnan(gamma).any())
    # a repeat needs a blank between: 2 2 does not fit in 2 frames, 2 3 does
    assert float(cpr.prefix_state(lp, 2, [2, 2], eos=None)[1]) == float('-inf')
    assert math.isfinite(float(cpr.prefix_state(lp, 2, [2, 3], eos=None)[1]))
    assert float(cpr.prefix_state(lp, 3, [2, 2])[1]) > float('-inf')
    # one frame: one label at most, and the completed sequence is that frame's log-prob
    g1, p1 = cpr.prefix_state(lp, 1, [3], eos=None)
    assert abs(float(p1) - float(lp[0, 3])) < 1e-12 and float(cpr.prefix_state(lp, 1, [3, 2], eos=None)[1]) == float('-inf')
    assert abs(float(cpr.prefix_state(lp, 1, [EOS])[1]) - float(lp[0, EOS])) < 1e-12
    # extending an impossible prefix, and extending by the blank: -inf throughout, no NaN
    for gam, empty, last in ((gamma, False, 4), (g1, False, 3)):
        g2, p2 = cpr.extend(lp, gam.shape[0], gam, empty, last, [0, 1, 2, 3, 4])
        assert not bool(torch.isnan(g2).any()) and not bool(torch.isnan(p2).any())
        assert float(p2[0]) == float('-inf') and bool(torch.isneginf(g2[0]).all())
    # the joint score of a -inf candidate under a -inf hypothesis is -inf
    s = cpr.JointSearch(lp[None], [1], beam=2, P=4, ctc_weight=0.5)
    att = torch.log_softmax(torch.randn(2, 5, generator=torch.Generator().manual_seed(1)), -1)
    for _ in range(3):
        s.step(att)
        assert not bool(torch.isnan(s.joint).any()) and not bool(torch.isnan(s.scores).any())


@pytest.mark.parametrize('with_lm', [False, True])
def test_weight_zero_is_the_plain_beam_step(with_lm):
    """ctc_weight 0 through JointSearch: ids and scores of oracle.beam_search.beam_step on the same inputs, every step."""
    B, beam, V, T, P = 3, 4, 50, 20, 8
    g = torch.Generator().manual_seed(11)
    lp = torch.stack([_lp(T, V, 20 + b) for b in range(B)])
    s = cpr.JointSearch(lp, [20, 13, 5], beam, P, ctc_weight=0.0, lm_weight=0.3 if with_lm else 0.0)
    preds, scores, flag = s.preds.clone(), s.scores.clone(), s.flag.clone()
    for step in range(6):
        att = torch.log_softmax(3 * torch.randn(B * beam, V, generator=g, dtype=torch.float64), -1)
        if step >= 2:
            att[:, EOS] += 2.0                                     # some hypotheses end, so the finished masking runs too
        lm = torch.log_softmax(torch.randn(B * beam, V, generator=g, dtype=torch.float64), -1) if with_lm else None
        s.step(att, lm)
        preds, scores, flag = beam_step(att, preds, scores, flag, beam, lm_log_probs=lm, lm_weight=0.3 if with_lm else 0.0)
        assert torch.equal(s.preds, preds) and torch.equal(s.flag, flag), step
        assert torch.equal(s.scores, scores), step
    assert bool(flag.any())


def test_the_ctc_term_changes_the_search():
    """Peaked CTC log-probs for y: the joint search at a high weight follows y against a flat attention decoder's order."""
    V, T, beam = 12, 16, 3
    y = [5, 5, 7, 3]
    lp = torch.full((T, V), -8.0, dtype=torch.float64)
    for t, v in enumerate([5, 0, 5, 0, 7, 0, 3, 0, EOS] + [0] * (T - 9)):
        lp[t, v] = 0.0
    lp = torch.log_softmax(lp, -1)
    att = torch.log_softmax(torch.linspace(0.0, 1.0, V, dtype=torch.float64), -1).expand(beam, V)
    s = cpr.JointSearch(lp[None], [T], beam, P=V, ctc_weight=0.9)
    for _ in range(len(y) + 1):
        s.step(att)
    best = s.preds[int(s.scores.view(-1).argmax())].tolist()
    assert best == [EOS] + y + [EOS]


# ------------------------------------------------------------------------------------------------ recognizer arguments
def _speech_params(ctc_weight):
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
            'frontend': dict(input_size=40, output_size=256, in_channel=1, mid_channel=8, out_channel=8,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=256, n_heads=4, d_ff=256, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.0, normalize_before=False, concat_after=False,
                            activation='glu', relative_positional=False),
            'decoder': dict(vocab_size=30, d_model=256, n_heads=4, d_ff=256, memory_dim=256, n_blocks=1, pos_dropout=0.0,
                            slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.0,
                            activation='glu', normalize_before=False, concat_after=False, share_embedding=True),
            'ctc_weight': ctc_weight, 'encoder_output_size': 256, 'smoothing': 0.1}


def test_recognizer_argument_checks():
    """All before any device work: the tensors stay on the CPU (ngpu = 0)."""
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.recognize import SpeechToTextRecognizer, build_recognizer
    joint, plain = SpeechToText(_speech_params(0.3)), SpeechToText(_speech_params(0.0))
    with pytest.raises(ValueError, match='needs the joint-CTC head'):
        SpeechToTextRecognizer(plain, ctc_weight=0.3, ngpu=0)
    for w in (-0.1, 1.5):
        with pytest.raises(ValueError, match=r'ctc_weight must be in \[0, 1\]'):
            SpeechToTextRecognizer(joint, ctc_weight=w, ngpu=0)
    for P in (4, 17):
        with pytest.raises(ValueError, match='ctc_candidates must be in'):
            SpeechToTextRecognizer(joint, ctc_weight=0.3, beam_width=5, ctc_candidates=P, ngpu=0)
    assert SpeechToTextRecognizer(joint, ctc_weight=0.3, beam_width=5, ngpu=0).ctc_candidates == 10
    assert SpeechToTextRecognizer(joint, ctc_weight=0.3, beam_width=10, ngpu=0).ctc_candidates == 16
    assert SpeechToTextRecognizer(joint, ctc_weight=0.3, beam_width=16, ctc_candidates=16, ngpu=0).ctc_candidates == 16
    SpeechToTextRecognizer(plain, ctc_weight=0.0, beam_width=5, ngpu=0)            # weight 0 needs no head
    with pytest.raises(ValueError, match='recognize_spans needs the joint-CTC head'):
        SpeechToTextRecognizer(plain, ngpu=0).recognize_spans(torch.zeros(1, 40, 40), torch.ones(1, 40, dtype=torch.bool))
    args = SimpleNamespace(lm_weight=0.1, ctc_weight=0.3, beam_width=5, nbest=1, max_len=20, penalty=0.6, lamda=5, ngpu=0,
                           ctc_candidates=12)
    rec = build_recognizer('speech2text', joint, None, args, None)
    assert rec.ctc_weight == 0.3 and rec.ctc_candidates == 12
    del args.ctc_candidates
    assert build_recognizer('speech2text', joint, None, args, None).ctc_candidates == 10


def test_decode_step_refuses_the_ctc_weight():
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.recognize import SpeechToTextRecognizer
    rec = SpeechToTextRecognizer(SpeechToText(_speech_params(0.3)), ctc_weight=0.3, beam_width=2, ngpu=0)
    preds = torch.ones(2, 1, dtype=torch.int64)
    with pytest.raises(NotImplementedError, match=r'recognize\(\)'):
        rec.decode_step(preds, torch.zeros(2, 9, 256), torch.ones(2, 9, dtype=torch.bool), {'decoder': None},
                        torch.zeros(2, 1), torch.zeros(2, 1, dtype=torch.bool))
