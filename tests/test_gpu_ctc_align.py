"""GPU checks of CTC forced alignment (otb_ctc_align): the kernel against torchaudio's forced_align and merge_tokens on the
same fp32 log-probs, against the CPU restatement (tests/ctc_align_ref.py) where torchaudio cannot say (batches with
infeasible rows, ties), the logit + log-sum-exp mode, consistency with the CTC loss and the greedy decoder, and the
model-level entry points (CTCModel.align, SpeechToText.align, CTCRecognizer.recognize_spans)."""
import numpy as np
import pytest
import torch

from tests import ctc_align_ref as car

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    from opentransformer_b200.recognize import CTCRecognizer
    DEV = torch.device('cuda:0')


def _lp(B, T, V, seed, scale=3.0):
    g = torch.Generator().manual_seed(seed)
    return torch.log_softmax(scale * torch.randn(B, T, V, generator=g), dim=-1)


def _batch(B, T, V, Ls, seed, tight=()):
    """Targets of the given lengths (with repeats) padded to max(Ls), and frame counts: a tight fit for the rows in
    `tight`, a random count between the fewest frames and T for the others (row 0 gets all T)."""
    g = torch.Generator().manual_seed(seed)
    toks = [car.tokens_with_repeats(L, V, g) for L in Ls]
    n = []
    for b, tk in enumerate(toks):
        lo = max(car.min_frames(tk), 1)
        assert lo <= T
        n.append(lo if b in tight else T if b == 0 else int(torch.randint(lo, T + 1, (), generator=g)))
    Lmax = max(Ls)
    tgt = torch.zeros(B, Lmax, dtype=torch.int64)
    for b, tk in enumerate(toks):
        tgt[b, :len(tk)] = torch.tensor(tk, dtype=torch.int64)
    return toks, torch.tensor(n, dtype=torch.int32), tgt, torch.tensor(Ls, dtype=torch.int32)


def _run(lp, n, tgt, tlen, lse=None):
    out = ops.ctc_align(lp.to(DEV), n.to(DEV), tgt.to(DEV), tlen.to(DEV), lse=None if lse is None else lse.to(DEV))
    return [t.cpu() for t in out]


def _check_row(b, got, lp_b, tokens, nb):
    labels, scores, spans, path = got
    ta_labels, ta_scores, ta_spans = car.torchaudio_align(lp_b[:nb], tokens)
    assert np.array_equal(labels[b, :nb].numpy(), ta_labels), b
    assert bool((labels[b, nb:] == -1).all()), b
    assert np.array_equal(scores[b, :nb].numpy().view(np.int32), ta_scores.view(np.int32)), b       # bit-identical
    L = len(tokens)
    assert np.array_equal(spans[b, :L].numpy(), ta_spans), b
    assert bool((spans[b, L:] == -1).all()), b
    want = float(np.add.accumulate(ta_scores.astype(np.float64))[-1]) if nb else 0.0
    assert abs(float(path[b]) - want) <= 1e-6 * max(1.0, abs(want)) + 2e-7 * nb, (b, float(path[b]), want)
    if nb:
        assert float(path[b]) == float(np.add.accumulate(ta_scores, dtype=np.float32)[-1]), b     # the same fp32 sums


# ------------------------------------------------------------------------------------------------ kernel vs torchaudio
CASES = {
    # name: (B, T, V, target lengths, rows aligned with a tight fit)
    'ragged32': (32, 400, 4234, [int(x) for x in torch.randint(0, 150, (32,), generator=torch.Generator().manual_seed(5))], (3, 7)),
    'L0': (3, 50, 40, [0, 0, 0], ()),
    'L1': (4, 30, 40, [1, 1, 1, 1], (1,)),
    'L64': (4, 200, 100, [64, 64, 10, 64], (2,)),
    'L65': (4, 200, 100, [65, 65, 65, 0], (1,)),
    'L300': (3, 1000, 4234, [300, 300, 299], (1,)),
    'L1023': (2, 1400, 4234, [1023, 1023], (1,)),
}


@pytest.mark.parametrize('case', list(CASES))
def test_kernel_matches_torchaudio(case):
    B, T, V, Ls, tight = CASES[case]
    toks, n, tgt, tlen = _batch(B, T, V, Ls, seed=len(case) + B, tight=tight)
    lp = _lp(B, T, V, seed=B * T)
    got = _run(lp, n, tgt, tlen)
    for b in range(B):
        _check_row(b, got, lp[b], toks[b], int(n[b]))


def test_infeasible_rows_leave_their_neighbours_alone():
    """Too few frames, a blank in the target, a token >= V, no frames for a non-empty target, tgt_len > Lmax: path score
    -inf, labels / spans -1, frame scores -inf; the feasible rows between them are aligned as alone."""
    B, T, V = 8, 60, 30
    toks, n, tgt, tlen = _batch(B, T, V, [20, 20, 10, 20, 12, 20, 20, 5], seed=3)
    lp = _lp(B, T, V, seed=9)
    n[1] = car.min_frames(toks[1]) - 1            # one frame short
    tgt[3, 4] = 0                                 # the blank inside a target
    tgt[5, 0] = V                                 # out of the vocabulary
    n[6] = 0                                      # no frames
    tlen[7] = tgt.shape[1] + 1                    # more tokens than the rows hold
    labels, scores, spans, path = got = _run(lp, n, tgt, tlen)
    for b in (1, 3, 5, 6, 7):
        assert float(path[b]) == float('-inf'), b
        assert bool((labels[b] == -1).all()) and bool((spans[b] == -1).all()) and bool(torch.isneginf(scores[b]).all()), b
    for b in (0, 2, 4):
        _check_row(b, got, lp[b], toks[b], int(n[b]))
    empty = _run(lp[:1], torch.tensor([0], dtype=torch.int32), tgt[:1, :0], torch.tensor([0], dtype=torch.int32))
    assert float(empty[3][0]) == 0.0 and bool((empty[0] == -1).all())


@pytest.mark.parametrize('seed', [0, 1])
def test_ties_match_the_restatement(seed):
    """Log-probs from a handful of values, so that many alignments tie: the kernel follows the restatement's tie-break."""
    B, T, V = 6, 80, 5
    toks, n, tgt, tlen = _batch(B, T, V, [0, 1, 7, 20, 30, 33], seed=seed, tight=(5,))
    g = torch.Generator().manual_seed(seed)
    lp = torch.randint(-3, 1, (B, T, V), generator=g).float()
    lp[0, :5] = 0.0                                 # whole frames of equal numbers
    got = _run(lp, n, tgt, tlen)
    for b in range(B):
        want = car.viterbi_align(lp[b], toks[b], n_frames=int(n[b]))
        assert np.array_equal(got[0][b].numpy(), want[0]), b
        assert np.array_equal(got[1][b].numpy(), want[1]), b
        assert np.array_equal(got[2][b, :len(toks[b])].numpy(), want[2]), b
        assert float(got[3][b]) == float(want[3]), b


def test_logit_mode_matches_log_prob_mode():
    """rows = logits with lse = each frame's log-sum-exp gives the labels of the log-prob mode on inputs where one
    alignment stands out, and scores within 1e-5."""
    B, T, V = 8, 150, 500
    toks, n, tgt, tlen = _batch(B, T, V, [40, 3, 0, 60, 25, 70, 1, 50], seed=21)
    g = torch.Generator().manual_seed(22)
    logits = torch.randn(B, T, V, generator=g) + 4.0
    for b in range(B):                       # lift a random alignment of each target by 6 nats per frame
        labels = car.viterbi_align(torch.log_softmax(torch.randn(T, V, generator=g), -1), toks[b], n_frames=int(n[b]))[0]
        for t, k in enumerate(labels.tolist()):
            if k >= 0:
                logits[b, t, k] += 6.0
    lse = torch.logsumexp(logits.double(), dim=-1).float()
    lp = (logits.double() - lse.double()[..., None]).float()
    a = _run(lp, n, tgt, tlen)
    c = _run(logits, n, tgt, tlen, lse=lse)
    assert torch.equal(a[0], c[0]) and torch.equal(a[2], c[2])
    valid = a[0] >= 0
    assert float((a[1][valid] - c[1][valid]).abs().max()) < 1e-5
    assert bool(torch.isneginf(c[1][~valid]).all())
    assert float(((a[3] - c[3]).abs() / a[3].abs().clamp_min(1.0)).max()) < 1e-5


# ------------------------------------------------------------------------------------------------ the other CTC kernels
def test_path_score_is_bounded_by_the_ctc_loss():
    """max over alignments <= log-sum over alignments: path score <= -nll of otb_ctc_loss, equal where T' = L and no token
    repeats (one alignment)."""
    B, T, V = 6, 100, 40
    g = torch.Generator().manual_seed(4)
    logits = (3.0 * torch.randn(B * T, (V + 7) // 8 * 8, generator=g)).to(DEV)
    toks, n, tgt, tlen = _batch(B, T, V, [64, 30, 1, 0, 35, 64], seed=8)
    for b in (1, 4):                                 # one alignment: T' = L distinct tokens
        toks[b] = [int(k) for k in torch.randperm(V - 1, generator=g)[:int(tlen[b])] + 1]
        tgt[b, :tlen[b]] = torch.tensor(toks[b])
        n[b] = tlen[b]
    lp = ops.log_softmax(logits, V).view(B, T, V)
    _, nll, _ = ops.ctc_loss(logits, B, T, V, n.to(DEV), tgt.to(DEV), tlen.to(DEV))
    _, _, _, path = ops.ctc_align(lp, n.to(DEV), tgt.to(DEV), tlen.to(DEV))
    nll, path = nll.cpu(), path.cpu()
    assert bool((path <= -nll + 1e-4 * nll.abs().clamp_min(1.0)).all()), (path, -nll)
    for b in (1, 4):
        assert abs(float(path[b]) + float(nll[b])) <= 1e-5 * abs(float(nll[b])), b


@pytest.mark.parametrize('B,T', [(1, 7), (32, 249)])
def test_greedy_path_is_its_own_alignment(B, T):
    """Aligning the greedy 1-best gives back the frame-wise argmax labels and the greedy score."""
    V = 40
    g = torch.Generator().manual_seed(B + T)
    best = torch.randint(0, 5, (B, T), generator=g)                # runs and repeats of a few tokens, blanks among them
    logits = torch.randn(B * T, V, generator=g)
    logits.view(B, T, V).scatter_add_(2, best.unsqueeze(2), torch.full((B, T, 1), 4.0))
    logits = logits.to(DEV)
    n = torch.randint(1, T + 1, (B,), generator=g).to(torch.int32)
    n[0] = T
    n = n.to(DEV)
    top_lp, top_id = ops.ctc_frame_topk(logits, B, T, V, n, 1)
    ids, nout, sc = ops.ctc_greedy(top_lp, top_id, B, T, n)
    lp = ops.log_softmax(logits, V).view(B, T, V)
    labels, _, _, path = ops.ctc_align(lp, n, ids, nout)
    valid = torch.arange(T, device=DEV)[None] < n[:, None]
    want = torch.where(valid, top_id.view(B, T), -1)
    assert torch.equal(labels, want)
    assert float(((path - sc).abs() / sc.abs().clamp_min(1.0)).max()) < 1e-5


# ------------------------------------------------------------------------------------------------ models
def _model_case(encoder_type):
    from tests.test_gpu_ctc_model import _batch as ctc_batch, _build, _params
    model, _ = _build(_params(encoder_type))
    x, mask, tgt, tlen = ctc_batch()
    return model, x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV)


def _check_against_torchaudio(out, lp, lengths, tokens_rows, n_tokens):
    labels, scores, spans, path = (t.cpu() for t in out)
    for b in range(lp.shape[0]):
        tk = tokens_rows[b, :int(n_tokens[b])].tolist()
        _check_row(b, (labels, scores, spans, path), lp[b].cpu(), tk, int(lengths[b]))


@pytest.mark.parametrize('encoder_type', ['transformer', 'conformer'])
def test_ctc_model_align(encoder_type):
    """CTCModel.align is torchaudio on CTCModel.inference's log-probs, targets as forward slices them; in train() it runs
    the same inference path."""
    model, x, mask, tgt, tlen = _model_case(encoder_type)
    model.eval()
    out = model.align(x, mask, tgt, tlen)
    with torch.no_grad():
        lp, lengths = model.inference(x, mask)
    _check_against_torchaudio(out, lp, lengths, tgt[:, 1:-1].cpu(), (tlen - 1).cpu())
    model.train()
    again = model.align(x, mask, tgt, tlen)
    assert all(torch.equal(a, b) for a, b in zip(out, again))


def test_speech_to_text_align():
    """SpeechToText.align through the joint-CTC head: torchaudio on the head's log-probs, targets[:, 1:] with
    targets_length tokens, as the joint CTC loss scores them."""
    from tests.test_gpu_train import _batch as speech_batch, _build as speech_build, _params as speech_params
    params = speech_params(n_enc=2, n_dec=1)
    params['ctc_weight'] = 0.3
    params['encoder_output_size'] = 256
    model, _ = speech_build(params)
    model.eval()
    x, mask, tgt = (t.to(DEV) for t in speech_batch())
    tlen = (tgt[:, 1:] != 0).sum(1)
    out = model.align(x, mask, tgt, tlen)
    with torch.no_grad():
        mem, lengths, B, T2 = model.encode_bf16(x, mask)
        V = model.decoder.vocab_size
        lp = ops.log_softmax(model.assistor.logits_bf16(mem), V).view(B, T2, V)
    _check_against_torchaudio(out, lp, lengths, tgt[:, 1:].cpu(), tlen.cpu())


@pytest.mark.parametrize('mode,beam', [('greedy', 1), ('beam', 10)])
def test_recognize_spans(mode, beam):
    """recognize_spans: the 1-best of recognize_ids, and the spans CTCModel.align gives for it."""
    model, x, mask, _, _ = _model_case('transformer')
    rec = CTCRecognizer(model, beam_width=beam, mode=mode)
    ids, n, sc = rec.recognize_ids(x, mask)
    ids2, n2, sc2, spans = rec.recognize_spans(x, mask)
    assert torch.equal(ids, ids2) and torch.equal(n, n2) and torch.equal(sc, sc2)
    B, T2 = ids.shape[0], ids.shape[2]
    truth = torch.zeros(B, T2 + 2, dtype=torch.int64, device=DEV)      # the collate's layout: <S/E> tokens <S/E>
    truth[:, 0] = 1
    truth[:, 1:T2 + 1] = ids[:, 0]
    truth[torch.arange(B, device=DEV), n[:, 0].long() + 1] = 1
    _, _, want, path = model.align(x, mask, truth, n[:, 0] + 1)
    assert torch.equal(spans, want[:, :spans.shape[1]])
    assert bool(torch.isfinite(path).all())
    for b in range(B):
        k = int(n[b, 0])
        assert bool((spans[b, :k] >= 0).all()) and bool((spans[b, k:] == -1).all())
