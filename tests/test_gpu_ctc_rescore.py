"""GPU checks of CTC rescoring of the attention n-best (DESIGN.md 4.18): otb_ctc_nbest_score against float64
F.ctc_loss per row (tests/ctc_rescore_ref.py) at ragged lengths and at the edges it defines, and the recognizer's
apply_ctc_rescoring end to end against the restatement run on its own first-pass n-best."""
import pytest
import torch

from tests import ctc_rescore_ref as cr
from tests import rescore_ref as rr

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    from opentransformer_b200 import recognize
    from opentransformer_b200.recognize import SpeechToTextRecognizer
    from tests.test_gpu_rescore import _inputs, _speech_model, _tol, _transformer_lm
    DEV = torch.device('cuda:0')

EOS, NEG_INF = rr.EOS, rr.NEG_INF
# fp32 log-domain accumulation: alpha_t grows to the final |log p| over T' frames and each step rounds once at that
# magnitude (2^-24 relative), plus log_add's absolute error of a few 1e-7 per frame: 1e-4 relative leaves ample margin at
# T' <= 1200; the absolute term covers scores near 0.
RTOL, ATOL = 1e-4, 1e-4


# ------------------------------------------------------------------------------------------------ otb_ctc_nbest_score
def _targets(B, K, V, row_lens, g, planted=True):
    """i32 [B, K, max(row_lens)]: random labels 2..V-1 closed by <S/E>, -1 after; with `planted`, runs of repeated labels,
    a blank label and an out-of-range label in some rows."""
    Lp = max(row_lens)
    tg = torch.full((B, K, Lp), -1, dtype=torch.int32)
    i = 0
    for b in range(B):
        for k in range(K):
            n = row_lens[i % len(row_lens)]
            y = torch.randint(2, V, (n,), generator=g, dtype=torch.int32)
            if planted and n > 3 and i % 3 == 1:
                y[1:n // 2] = y[0]                                  # a run of repeats: needs a blank between each
            if planted and n > 2 and i % 7 == 5:
                y[n // 2] = 0                                       # the blank as a label
            if planted and n > 2 and i % 11 == 8:
                y[n // 3] = V                                       # out of range
            y[-1] = EOS
            tg[b, k, :n] = y
            i += 1
    return tg


def _check_kernel(B, K, T, V, in_len, row_lens, seed, planted=True, pad_cols=0):
    g = torch.Generator().manual_seed(seed)
    logits = 3.0 * torch.randn(B * T, V, generator=g)
    logp = torch.log_softmax(logits, -1)
    tg = _targets(B, K, V, row_lens, g, planted)
    il = torch.tensor(in_len, dtype=torch.int32)
    full = torch.full((B * T, V + pad_cols), float('nan'), device=DEV)     # pad columns must not be read
    full[:, :V] = logp.to(DEV)
    got = ops.ctc_nbest_score(full[:, :V], B, T, il.to(DEV), tg.to(DEV)).double().cpu()
    want = cr.nbest_scores(logp, B, T, il, tg)
    inf_got, inf_want = torch.isinf(got), torch.isinf(want)
    assert torch.equal(inf_got, inf_want), (inf_got, inf_want)
    assert bool((got[inf_got] == NEG_INF).all()) and not bool(torch.isnan(got).any())
    fin = ~inf_want
    err = float(((got - want).abs() / (want.abs() * RTOL + ATOL))[fin].max()) if bool(fin.any()) else 0.0
    print(f'ctc_nbest_score B {B} K {K} T {T} Lp {tg.shape[2]}: {int(fin.sum())} finite rows, {int(inf_want.sum())} -inf, '
          f'worst error / tolerance {err:.3f}')
    assert err <= 1.0
    return want


@pytest.mark.parametrize('K', [1, 5, 16])
def test_short_rows_ragged_frames_and_edges(K):
    """Ragged in_len including 0 and 1, rows of 1..14 labels with repeats, blank and out-of-range labels, rows too long
    for their utterance."""
    B, T, V = 6, 40, 50
    want = _check_kernel(B, K, T, V, [40, 17, 0, 33, 1, 9], list(range(1, 15)), seed=K, pad_cols=12)
    assert bool(torch.isinf(want[2]).all())                         # in_len 0
    assert bool(torch.isfinite(want).any()) and bool(torch.isinf(want[[0, 1, 3, 4, 5]]).any())


@pytest.mark.parametrize('L', [1, 63, 64, 65, 159, 160])
def test_label_widths_around_the_launch_shapes(L):
    """One label (just <S/E>) and the row widths on either side of the 128- and 320-state instances."""
    B, K, T, V = 3, 4, 2 * L + 40, 60
    _check_kernel(B, K, T, V, [T, T - 7, L + 3], [L, max(1, L - 1), max(1, L // 2)], seed=L)


@pytest.mark.parametrize('L', [1023, 1024])
def test_the_longest_rows_a_recognizer_produces(L):
    """max_len 1023 tokens and the closing <S/E>: S up to 2049 states."""
    B, K, V = 2, 3, 60
    T = L + 120
    want = _check_kernel(B, K, T, V, [T, L + 30], [L, L - 1, 400], seed=L, planted=False)
    assert bool(torch.isfinite(want[0]).all())


def test_one_frame_per_label_and_no_more():
    """A row of n distinct labels needs n frames; with n - 1 it has no alignment.  Repeats need one frame more each."""
    B, K, T, V = 1, 3, 8, 20
    logp = torch.log_softmax(torch.randn(B * T, V), -1)
    tg = torch.tensor([[[2, 3, 4, 5, 6, 7, 8, 1], [2, 3, 4, 5, 6, 7, 8, 9], [2, 2, 3, 4, 5, 6, 7, 1]]], dtype=torch.int32)
    for n in (8, 7):
        il = torch.tensor([n], dtype=torch.int32)
        got = ops.ctc_nbest_score(logp.to(DEV), B, T, il.to(DEV), tg.to(DEV)).cpu()
        want = cr.nbest_scores(logp, B, T, il, tg)
        assert torch.equal(torch.isinf(got), torch.isinf(want))
    assert torch.isinf(got).all()                                   # 7 frames: none of the three fits


# ------------------------------------------------------------------------------------------------ the recognizer
def _ctc_second(model, mem, mem_len, T2):
    """The head's float64 log-probs on the port's memory with the bf16 weights the port multiplies by -> (b, y) -> the CTC
    score of y <S/E>."""
    head = model.assistor.output_layer
    memory = mem.double().cpu()
    logits = memory @ head.weight.detach().to(torch.bfloat16).double().cpu().t() + head.bias.detach().double().cpu()
    logp = torch.log_softmax(logits, -1).view(-1, T2, logits.shape[1])
    return lambda b, y: cr.ctc_score(logp[b, :int(mem_len[b])], list(y) + [EOS])


def _check(ids, scores, hyps, s1, ctc_of, others_of, weight, nbest):
    """tests/test_gpu_rescore's comparison with the CTC re-ranking rule: per utterance the port's n-best against
    ctc_rescore_ref.rerank on the same first-pass hypotheses."""
    B = len(hyps)
    lens = (torch.cat((ids, torch.full((B, ids.shape[1], 1), EOS, dtype=ids.dtype)), 2) == EOS).int().argmax(dim=2)
    for b in range(B):
        ref = cr.rerank(hyps[b], s1[b], [others_of(b, y) for y in hyps[b]], [ctc_of(b, y) for y in hyps[b]], weight,
                        len(hyps[b]))
        key = lambda y, s: (tuple(y), s != NEG_INF)
        port = [(ids[b, i, :int(lens[b, i])].tolist(), float(scores[b, i])) for i in range(nbest)]
        ref_s = {key(y, s): s for _, y, s in ref}
        for y, s in port:
            assert key(y, s) in ref_s, (b, y)
            r = ref_s[key(y, s)]
            assert (s == NEG_INF) == (r == NEG_INF) and (r == NEG_INF or abs(s - r) <= _tol(r)), (b, y, s, r)
        for i in range(nbest):
            gap = ref[i][2] - ref[i + 1][2] if i + 1 < len(ref) else float('inf')
            if gap > _tol(ref[i][2]):
                assert {key(y, s) for y, s in port[:i + 1]} == {key(y, s) for _, y, s in ref[:i + 1]}, (b, i)


def _run(model, x, mask, beam, nbest, L, w, lm=None, **kw):
    """apply_ctc_rescoring's result, the first pass it started from and the same search without the flag."""
    common = dict(beam_width=beam, max_len=L, penalty=0.6, lamda=5, **kw)
    rec = SpeechToTextRecognizer(model, lm=lm, nbest=nbest, apply_ctc_rescoring=True, apply_lm_rescoring=lm is not None,
                                 rescore_weight=w, **common)
    ids, scores, steps = rec.recognize_ids(x, mask)
    bd = next(iter(rec._decoders.values()))
    first, first_sc = bd.state.finalize(0.6, 5, beam)
    p0, s0, n0 = SpeechToTextRecognizer(model, nbest=beam, **common).recognize_ids(x, mask)
    assert n0 == steps and torch.equal(first[:, :, :steps], p0) and torch.equal(first_sc, s0)     # the search is unchanged
    assert ids.shape == (x.shape[0], nbest, steps)
    return rec, bd, ids, scores, steps, p0, s0


@pytest.mark.parametrize('nbest,with_lm', [(1, False), (4, False), (3, True)])
def test_ctc_rescoring_of_the_persistent_first_pass(nbest, with_lm):
    """The search runs on the persistent kernel (no per-step graph was captured), then the head re-ranks its beam_width
    hypotheses; with apply_lm_rescoring the LM and the CTC score add before the weight."""
    model, _, _ = _speech_model(ctc_weight=0.3, eos_bias=0.0)
    B, beam, L, w = 4, 6, 24, 0.6
    x, mask = _inputs(B, 400, [400, 377, 250, 181], seed=4)
    lm, lm_second = _transformer_lm(model.decoder.vocab_size) if with_lm else (None, None)
    rec, bd, ids, scores, steps, p0, s0 = _run(model, x, mask, beam, nbest, L, w, lm=lm)
    assert bd.persistent and bd.graph is None and bd.ctc is None
    with torch.no_grad():
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
    hyps = [[rr.cut(p0[b, k].tolist()) for k in range(beam)] for b in range(B)]
    others = (lambda b, y: [lm_second(b, y)]) if with_lm else (lambda b, y: [])
    _check(ids.cpu(), scores.cpu(), hyps, s0.cpu().tolist(), _ctc_second(model, mem, mem_len, T2), others, w, nbest)


def test_an_utterance_without_alignments_keeps_its_first_pass_order():
    """No <S/E> (every hypothesis runs to max_len 40) and an utterance of ~24 encoder frames: none of its 41-label rows fits,
    so its n-best is the first pass's, scored -inf; the other utterance is re-ranked."""
    model, _, _ = _speech_model(ctc_weight=0.3)
    B, beam, nbest, L, w = 2, 5, 5, 40, 1.0
    x, mask = _inputs(B, 400, [400, 100], seed=6)
    rec, bd, ids, scores, steps, p0, s0 = _run(model, x, mask, beam, nbest, L, w)
    assert bd.persistent and int(bd.mem_len[1]) < L + 1
    assert torch.equal(ids[1], p0[1]) and bool((scores[1] == NEG_INF).all())
    assert bool(torch.isfinite(scores[0]).any())


def test_recognize_spans_aligns_the_rescored_best():
    from opentransformer_b200.model import ctc_align_logits
    model, _, _ = _speech_model(ctc_weight=0.3, eos_bias=0.0)
    B = 3
    x, mask = _inputs(B, 240, [240, 200, 131], seed=2)
    rec = SpeechToTextRecognizer(model, beam_width=6, nbest=2, max_len=30, apply_ctc_rescoring=True, rescore_weight=0.7)
    ids, scores, steps, spans = rec.recognize_spans(x, mask)
    ids2, scores2, steps2 = rec.recognize_ids(x, mask)
    assert steps == steps2 and torch.equal(ids, ids2) and torch.equal(scores, scores2)
    with torch.no_grad():
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
        best = torch.cat((ids[:, 0], torch.full((B, 1), EOS, dtype=ids.dtype, device=DEV)), dim=1)
        n_tok = (best == EOS).int().argmax(dim=1) + 1
        want = ctc_align_logits(model.assistor.logits_bf16(mem), mem_len, B, T2, model.decoder.vocab_size, best, n_tok, 0)[2]
    assert torch.equal(spans, want)


def test_conformer_decoder_384_on_the_per_step_path():
    """d_model 384 / 4 heads (the shipped Conformer configuration) is outside the persistent kernel: the per-step graph
    path's n-best is re-ranked the same way."""
    from tests.test_gpu_head_dim_96 import _build, _conformer_params
    params = _conformer_params(n_enc=1, n_dec=2)
    params['ctc_weight'] = 0.3
    params['encoder_output_size'] = params['encoder']['d_model']
    model, _ = _build(params)
    with torch.no_grad():
        model.decoder.output_layer.bias[1] = 0.0
    B, beam, nbest, L, w = 3, 5, 3, 20, 0.8
    x, mask = _inputs(B, 300, [300, 211, 250], seed=3)
    rec, bd, ids, scores, steps, p0, s0 = _run(model, x, mask, beam, nbest, L, w)
    assert not bd.persistent and bd.graph is not None
    with torch.no_grad():
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
    hyps = [[rr.cut(p0[b, k].tolist()) for k in range(beam)] for b in range(B)]
    _check(ids.cpu(), scores.cpu(), hyps, s0.cpu().tolist(), _ctc_second(model, mem, mem_len, T2), lambda b, y: [], w, nbest)


def test_flag_off_runs_no_new_code(monkeypatch):
    """Without apply_ctc_rescoring neither the kernel nor the recognizer's CTC term is reached, with or without LM
    rescoring, and the plain search returns what the rescoring recognizer's first pass holds."""
    model, _, _ = _speech_model(ctc_weight=0.3, eos_bias=0.0)
    B, beam, L = 3, 4, 16
    x, mask = _inputs(B, 300, [300, 260, 190], seed=5)
    on = SpeechToTextRecognizer(model, beam_width=beam, nbest=beam, max_len=L, apply_ctc_rescoring=True)
    on.recognize_ids(x, mask)
    first, first_sc = next(iter(on._decoders.values())).state.finalize(0, 5, beam)

    def new_code(*a, **k):
        raise AssertionError('CTC rescoring ran with the flag off')
    monkeypatch.setattr(ops, 'ctc_nbest_score', new_code)
    monkeypatch.setattr(recognize, 'ctc_rescoring_terms', new_code)
    ids, scores, steps = SpeechToTextRecognizer(model, beam_width=beam, nbest=beam, max_len=L).recognize_ids(x, mask)
    assert torch.equal(ids, first[:, :, :steps]) and torch.equal(scores, first_sc)
    lm, _ = _transformer_lm(model.decoder.vocab_size)
    SpeechToTextRecognizer(model, lm=lm, beam_width=beam, nbest=2, max_len=L, apply_lm_rescoring=True).recognize_ids(x, mask)
