"""CPU checks of n-best rescoring (DESIGN.md 4.10): the float64 restatement (tests/rescore_ref.py) against
F.cross_entropy and hand-built cases, the second pass's rows as the recognizers build them, the recognizers' refusals and
build_recognizer's plumbing.  No GPU: models stay on the CPU (ngpu = 0)."""
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from tests import rescore_ref as rr

EOS, NEG_INF = rr.EOS, rr.NEG_INF


@pytest.mark.parametrize('n', [0, 1, 5, 30])
def test_sequence_score_is_minus_the_summed_cross_entropy(n):
    g = torch.Generator().manual_seed(n)
    V = 40
    y = torch.randint(2, V, (n,), generator=g).tolist()
    logits = 3.0 * torch.randn(n + 4, V, generator=g, dtype=torch.float64)      # rows past n + 1 are padding: not read
    want = -F.cross_entropy(logits[:n + 1], torch.tensor(y + [EOS]), reduction='sum')
    got = rr.token_logprobs(logits, y)
    assert got.shape == (n + 1,)
    torch.testing.assert_close(rr.combine(0.0, [got], 1.0), want, rtol=0, atol=1e-12)


def test_cut():
    assert rr.cut([5, 6, EOS, 7, EOS]) == [5, 6]
    assert rr.cut([5, 6, 7]) == [5, 6, 7]                  # reached max_len: the <S/E> is implied
    assert rr.cut([EOS, 5]) == []
    assert rr.cut([5, 6, EOS, 0, 0], length=3) == [5, 6]   # a CTC row that emitted the closing <S/E> as a label
    assert rr.cut([5, 6, 9, 0, 0], length=2) == [5, 6]


def _tl(*vals):
    return [torch.tensor(vals, dtype=torch.float64)]


def test_rerank_drops_duplicates_keeps_ties_in_order_and_pads():
    hyps = [[5, 6], [5], [5, 6], [7], [5]]
    s1 = [-1.0, -2.0, -1.5, -3.0, -2.5]
    tok = [_tl(-1.0, -1.0, -1.0), _tl(-0.5, -0.5), _tl(-9.0, -9.0, -9.0), _tl(-0.25, -0.25), _tl(0.0, 0.0)]
    got = rr.rerank(hyps, s1, tok, 1.0, 5)
    # s: k0 -4, k1 -3, k2 dropped (= k0), k3 -3.5, k4 dropped (= k1)
    assert [(k, y) for k, y, _ in got] == [(1, [5]), (3, [7]), (0, [5, 6]), (None, []), (None, [])]
    assert [s for _, _, s in got] == [-3.0, -3.5, -4.0, NEG_INF, NEG_INF]
    ids, lens, sc = rr.as_tensors(got, 4)
    assert ids.tolist() == [[5, EOS, EOS, EOS], [7, EOS, EOS, EOS], [5, 6, EOS, EOS], [EOS] * 4, [EOS] * 4]
    assert lens.tolist() == [1, 1, 2, 0, 0]
    # equal s: the first-pass order decides
    tie = rr.rerank([[2], [3], [4]], [-1.0, -0.5, -1.0], [_tl(-1.0, 0.0), _tl(-1.5, 0.0), _tl(-1.0, 0.0)], 1.0, 2)
    assert [k for k, _, _ in tie] == [0, 1]
    # the nbest cut
    assert len(rr.rerank(hyps, s1, tok, 1.0, 2)) == 2


def test_weight_zero_is_the_first_pass_minus_duplicates():
    g = torch.Generator().manual_seed(3)
    hyps = [[4, 5], [4], [4, 5], [6, 7, 8], [9]]
    s1 = sorted(torch.randn(5, generator=g).tolist(), reverse=True)            # the first pass ranks its n-best
    tok = [[torch.randn(len(y) + 1, generator=g, dtype=torch.float64)] for y in hyps]
    got = rr.rerank(hyps, s1, tok, 0.0, 5)
    assert [k for k, _, _ in got] == [0, 1, 3, 4, None]
    assert [s for _, _, s in got[:4]] == [s1[0], s1[1], s1[3], s1[4]]


def test_models_add_before_the_weight():
    s = rr.combine(-2.0, [torch.tensor([-1.0, -2.0]), torch.tensor([-0.5])], 0.5)
    assert float(s) == -2.0 + 0.5 * (-3.0 - 0.5)


def test_second_pass_rows():
    """What the recognizers feed the second pass: BOS y PAD... / y <S/E> -1... / n, from attention rows (<S/E> after the end,
    or none at max_len) and from CTC rows (0 after the length, <S/E> possibly emitted)."""
    from opentransformer_b200.recognize import second_pass_rows
    att = torch.tensor([[[5, 6, EOS, EOS], [7, 8, 9, 10]], [[EOS, EOS, EOS, EOS], [4, EOS, EOS, EOS]]])
    inputs, tgt, n, Lp = second_pass_rows(att)
    assert Lp == 5 and n.tolist() == [[2, 4], [0, 1]]
    assert tgt.dtype == torch.int32 and inputs.dtype == torch.int64
    assert tgt.tolist() == [[[5, 6, EOS, -1, -1], [7, 8, 9, 10, EOS]], [[EOS, -1, -1, -1, -1], [4, EOS, -1, -1, -1]]]
    assert inputs.view(2, 2, 5).tolist() == [[[1, 5, 6, 1, 0], [1, 7, 8, 9, 10]], [[1, 1, 0, 0, 0], [1, 4, 1, 0, 0]]]
    ctc = torch.tensor([[[5, 6, EOS, 0, 0], [5, 6, 0, 0, 0], [0, 0, 0, 0, 0]]])
    inputs, tgt, n, Lp = second_pass_rows(ctc, torch.tensor([[3, 2, 0]]))
    assert Lp == 3 and n.tolist() == [[2, 2, 0]]
    assert tgt.tolist() == [[[5, 6, EOS], [5, 6, EOS], [EOS, -1, -1]]]
    for b in range(ctc.shape[0]):
        for k in range(ctc.shape[1]):
            assert rr.cut(ctc[b, k], [3, 2, 0][k]) == tgt[b, k, :n[b, k]].tolist()


# ------------------------------------------------------------------------------------------------ recognizer arguments
def _speech(ctc_weight, V=30):
    from opentransformer_b200.model import SpeechToText
    from tests.test_ctc_prefix_ref import _speech_params
    p = _speech_params(ctc_weight)
    p['decoder']['vocab_size'] = V
    return SpeechToText(p)


def _tlm(V=30):
    from opentransformer_b200.lm import TransformerLanguageModel
    return TransformerLanguageModel(dict(type='transformer_lm', vocab_size=V, num_blocks=1, d_model=256, n_heads=4, d_ff=256,
                                         residual_dropout=0.0, smoothing=0.1, share_embedding=True))


def _ctc_model(V=30):
    from opentransformer_b200.model import CTCModel
    from tests.test_ctc_prefix_ref import _speech_params
    p = _speech_params(0.0)
    p['vocab_size'] = V
    return CTCModel(p)


def test_refusals_before_any_device_work():
    from opentransformer_b200.recognize import CTCRecognizer, SpeechToTextRecognizer
    joint, plain, lm = _speech(0.3), _speech(0.0), _tlm()
    with pytest.raises(ValueError, match='apply_rescoring needs the joint-CTC head'):
        SpeechToTextRecognizer(plain, apply_rescoring=True, ngpu=0)
    with pytest.raises(ValueError, match='two uses of the joint-CTC head'):
        SpeechToTextRecognizer(joint, ctc_weight=0.3, apply_rescoring=True, ngpu=0)
    with pytest.raises(NotImplementedError, match='beam_width 1..16'):
        SpeechToTextRecognizer(joint, apply_rescoring=True, beam_width=17, ngpu=0)
    with pytest.raises(ValueError, match='apply_lm_rescoring needs an lm'):
        SpeechToTextRecognizer(plain, apply_lm_rescoring=True, ngpu=0)
    with pytest.raises(ValueError, match='one vocabulary'):
        SpeechToTextRecognizer(plain, lm=_tlm(31), apply_lm_rescoring=True, ngpu=0)
    with pytest.raises(ValueError, match='apply_lm_rescoring needs an lm'):
        CTCRecognizer(_ctc_model(), mode='beam', apply_lm_rescoring=True, ngpu=0)
    with pytest.raises(ValueError, match='one vocabulary'):
        CTCRecognizer(_ctc_model(), lm=_tlm(31), mode='beam', apply_lm_rescoring=True, ngpu=0)
    with pytest.raises(ValueError, match="use mode='beam'"):
        CTCRecognizer(_ctc_model(), lm=lm, mode='greedy', apply_lm_rescoring=True, ngpu=0)
    # accepted: every flag with what it needs
    rec = SpeechToTextRecognizer(joint, lm=lm, apply_rescoring=True, apply_lm_rescoring=True, rescore_weight=0.5,
                                 beam_width=16, ngpu=0)
    assert rec.apply_rescoring and rec.apply_lm_rescoring and rec.rescore_weight == 0.5
    assert not rec._lm_fused()
    assert SpeechToTextRecognizer(plain, lm=lm, ngpu=0)._lm_fused()             # the default: shallow fusion, as before
    assert CTCRecognizer(_ctc_model(), lm=lm, mode='beam', apply_lm_rescoring=True, ngpu=0).apply_lm_rescoring


def test_build_recognizer_plumbing():
    from opentransformer_b200.recognize import build_recognizer
    joint, lm = _speech(0.3), _tlm()
    args = SimpleNamespace(lm_weight=0.1, ctc_weight=0.0, beam_width=5, nbest=1, max_len=20, penalty=0.6, lamda=5, ngpu=0)
    rec = build_recognizer('speech2text', joint, None, args, None)                # fields absent: the defaults
    assert (rec.apply_rescoring, rec.apply_lm_rescoring, rec.rescore_weight) == (False, False, 1.0)
    args.apply_rescoring, args.apply_lm_rescoring, args.rescore_weight = True, True, 0.3
    rec = build_recognizer('speech2text', joint, lm, args, None)
    assert (rec.apply_rescoring, rec.apply_lm_rescoring, rec.rescore_weight) == (True, True, 0.3)
    cargs = SimpleNamespace(lm_weight=0.1, ngram_lm=None, beam_width=5, ngpu=0, mode='beam', alpha=0.1, beta=0.0)
    crec = build_recognizer('ctc', _ctc_model(), lm, cargs, None)
    assert (crec.apply_lm_rescoring, crec.rescore_weight) == (False, 1.0)
    cargs.apply_lm_rescoring, cargs.rescore_weight = True, 2.0
    crec = build_recognizer('ctc', _ctc_model(), lm, cargs, None)
    assert (crec.apply_lm_rescoring, crec.rescore_weight) == (True, 2.0)
    cargs.apply_rescoring = True
    with pytest.raises(ValueError, match='a CTC model has none'):
        build_recognizer('ctc', _ctc_model(), lm, cargs, None)
