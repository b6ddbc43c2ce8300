"""LM shallow fusion in the CTC prefix beam search on the GPU (DESIGN.md 4.19), with the Transformer and the recurrent LM:
weight 0 against otb_ctc_prefix_beam, a context-free LM against the fp32 restatement, random LMs against the restatement
over full-prefix LM calls, the LM's effect, graph against eager, recapture, and the recognizer's fused path with spans.
Small random models (vocab 40), ragged lengths with a 1-frame utterance, beam 1, 4 and 16."""
import pytest
import torch

from opentransformer_b200 import ops
from opentransformer_b200.ctc_fusion import CTCFusedSearch
from tests import ctc_lm_fusion_ref as fr

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda')
V, K, T = 40, 40, 12
LENS = [12, 1, 7, 10]
B = len(LENS)


def _lm(kind, seed, exact=False, bias=None):
    """A random LM with an untied output layer at its default initialisation (log-probs that move by tenths of a nat with
    the context); exact: output weight 0 and a random (or given) bias, so its log-probs are context-free and every path
    computes them exactly."""
    from opentransformer_b200.lm import RecurrentLanguageModel, TransformerLanguageModel
    torch.manual_seed(seed)
    if kind == 'transformer':
        lm = TransformerLanguageModel(dict(type='transformer_lm', vocab_size=V, num_blocks=2, d_model=256, n_heads=4, d_ff=256,
                                           residual_dropout=0.0, smoothing=0.1, share_embedding=False))
    else:
        lm = RecurrentLanguageModel(dict(vocab_size=V, share_embedding=False, smoothing=0.1, num_layers=2, hidden_size=64,
                                         dropout=0.0))
    if exact:
        with torch.no_grad():
            lm.output_project.weight.zero_()
            lm.output_project.bias.copy_(bias if bias is not None else 2.0 * torch.randn(V))
    return lm.to(DEV).eval()


def _frames(seed, boost=None):
    g = torch.Generator().manual_seed(seed)
    logits = 3.0 * torch.randn(B * T, V, generator=g)
    if boost is None:
        logits[:, 0] += 1.5
    else:
        logits[:, boost] += 8.0
    in_len = torch.tensor(LENS, dtype=torch.int32, device=DEV)
    lp, tok = ops.ctc_frame_topk(logits.to(DEV).contiguous(), B, T, V, in_len, K)
    lp_c, tok_c = lp.cpu(), tok.cpu()
    frames = [[[(int(tok_c[b * T + t, k]), lp_c[b * T + t, k].item()) for k in range(K) if tok_c[b * T + t, k] >= 0]
               for t in range(LENS[b])] for b in range(B)]
    return lp, tok, in_len, frames


def _nbest(out, b, W):
    ids, n, sc = (x.cpu() for x in out)
    return [(tuple(ids[b, s, :n[b, s]].tolist()), sc[b, s].item()) for s in range(W) if sc[b, s] > float('-inf')]


def _full_row(lm, P, memo):
    """log p_lm(. | <S/E> P) from the whole prefix: the uncached path (predict without a cache)."""
    if P not in memo:
        x = torch.tensor([[1] + list(P)], dtype=torch.int64, device=DEV)
        if lm.model_type == 'transformer_lm':
            row = lm.predict(x, last_frame=True)[0, 0]
        else:
            row = lm.predict(x)[0][0, -1]
        memo[P] = row.float().cpu().numpy()
    return memo[P]


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
@pytest.mark.parametrize('W', [1, 4, 16])
def test_weight_zero_is_bit_identical_to_the_unfused_search(kind, W):
    lm = _lm(kind, 1)
    lp, tok, in_len, _ = _frames(11)
    ids0, n0, sc0 = ops.ctc_prefix_beam(lp, tok, B, T, in_len, W)
    ids, n, sc = CTCFusedSearch(lm, B, W, T, K, DEV, 0.0, 0.0).run(lp, tok, in_len)
    assert torch.equal(ids, ids0.long()) and torch.equal(n, n0) and torch.equal(sc, sc0)


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
@pytest.mark.parametrize('W', [1, 4, 16])
def test_context_free_lm_matches_the_restatement(kind, W):
    """Ids exactly; scores within 1e-5 (1 + |s|): the restatement runs the kernel's fp32 sums, and exp / log1p may differ by
    an ulp in each of the 12 frames' log-adds."""
    lm = _lm(kind, 2, exact=True)
    row = _full_row(lm, (), {})
    lw, beta = 0.8, 0.3
    lp, tok, in_len, frames = _frames(12)
    out = CTCFusedSearch(lm, B, W, T, K, DEV, lw, beta).run(lp, tok, in_len)
    for b in range(B):
        want = fr.fused_prefix_beam_search(frames[b], W, lambda P: row, lw, beta, fp32=True)
        got = _nbest(out, b, W)
        assert [P for P, _ in got] == [P for P, _ in want], b
        for (_, s), (_, r) in zip(got, want):
            assert abs(s - r) <= 1e-5 * (1 + abs(r)), (b, s, r)


def _recreated_at_same_length(trace):
    """Frames where a slot is re-created by an extension at the length of the prefix it held, which survives in another
    slot: the case that rules out a [position, row] K/V layout."""
    hits = 0
    for prev, cur in zip(trace, trace[1:]):
        alive = {P for P, _ in cur}
        for s, (P, ext) in enumerate(cur):
            if ext and s < len(prev) and len(prev[s][0]) == len(P) and prev[s][0] != P and prev[s][0] in alive:
                hits += 1
    return hits


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
@pytest.mark.parametrize('W', [1, 4, 16])
def test_context_lm_matches_the_restatement_over_full_prefixes(kind, W):
    """The restatement's LM is predict on the whole prefix.  delta = lw * dev * (T + 1) + 1e-4, dev the largest
    |cached - full| LM log-prob of the final slots' prefixes measured here; scores of common prefixes agree within delta,
    and the 1-best agrees wherever the restatement's best two are more than delta apart."""
    lm = _lm(kind, 3)
    lw, beta = 0.6, 0.2
    memo, hazards, compared = {}, 0, 0
    for seed in range(3):
        lp, tok, in_len, frames = _frames(20 + seed)
        search = CTCFusedSearch(lm, B, W, T, K, DEV, lw, beta)
        out = search.run(lp, tok, in_len)
        rows = search.lm_rows.cpu().numpy()
        dev = 0.0
        for b in range(B):
            for s, (P, _) in enumerate(_nbest(out, b, W)):
                if len(P) < T:
                    dev = max(dev, float(abs(rows[b * W + s] - _full_row(lm, P, memo)).max()))
        assert dev < 0.05                       # bf16 rounding of two kernel paths, not a different context
        delta = lw * dev * (T + 1) + 1e-4
        for b in range(B):
            trace = []
            want = fr.fused_prefix_beam_search(frames[b], W, lambda P: _full_row(lm, P, memo), lw, beta, trace=trace)
            hazards += _recreated_at_same_length(trace)
            got = _nbest(out, b, W)
            if len(want) < 2 or want[0][1] - want[1][1] > delta:
                assert got[0][0] == want[0][0], (seed, b)
                compared += 1
            ref = dict(want)
            for P, s in got:
                if P in ref:
                    assert abs(s - ref[P]) <= delta, (seed, b, P, s, ref[P], delta)
    assert compared > 0
    if W > 1:
        assert hazards > 0


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_a_token_the_lm_rules_out_leaves_the_nbest(kind):
    X = 5
    bias = torch.zeros(V)
    bias[X] = -30.0
    lm = _lm(kind, 4, exact=True, bias=bias)
    lp, tok, in_len, _ = _frames(30, boost=X)
    ids0, n0, _ = ops.ctc_prefix_beam(lp, tok, B, T, in_len, 4)
    for b in range(B):
        if LENS[b] >= 7:
            assert X in ids0[b, 0, :n0[b, 0]].tolist()
    ids, n, sc = CTCFusedSearch(lm, B, 4, T, K, DEV, 10.0, 0.0).run(lp, tok, in_len)
    for b in range(B):
        for s in range(4):
            if sc[b, s] > float('-inf'):
                assert X not in ids[b, s, :n[b, s]].tolist(), (b, s)


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_graph_and_eager_agree_and_a_new_pack_recaptures(kind):
    lm = _lm(kind, 5)
    lp, tok, in_len, _ = _frames(40)
    g = CTCFusedSearch(lm, B, 4, T, K, DEV, 0.5, 0.2, use_graph=True)
    e = CTCFusedSearch(lm, B, 4, T, K, DEV, 0.5, 0.2, use_graph=False)
    r1, r2 = g.run(lp, tok, in_len), e.run(lp, tok, in_len)
    assert all(torch.equal(a, b) for a, b in zip(r1, r2))
    graph = g.graph
    assert all(torch.equal(a, b) for a, b in zip(g.run(lp, tok, in_len), r1)) and g.graph is graph
    lm.load_state_dict(_lm(kind, 6).state_dict())
    r3 = g.run(lp, tok, in_len)
    assert g.graph is not graph
    assert all(torch.equal(a, b) for a, b in zip(r3, e.run(lp, tok, in_len)))
    assert not torch.equal(r3[2], r1[2])


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_recognizer_fused_path_and_spans(kind):
    from opentransformer_b200.model import ctc_align_logits
    from opentransformer_b200.recognize import CTCRecognizer
    from tests.test_rescore_ref import _ctc_model
    torch.manual_seed(7)
    model = _ctc_model(V)
    lm = _lm(kind, 8)
    rec = CTCRecognizer(model, lm=lm, lm_weight=0.5, beta=0.2, beam_width=4, mode='beam', lm_fusion=True)
    x = torch.randn(2, 100, 40, device=DEV)
    mask = torch.ones(2, 100, dtype=torch.bool, device=DEV)
    mask[1, 60:] = False
    ids, n, sc = rec.recognize_ids(x, mask)
    ids2, n2, sc2, spans = rec.recognize_spans(x, mask)
    assert torch.equal(ids, ids2) and torch.equal(n, n2) and torch.equal(sc, sc2)
    with torch.no_grad():
        logits, lengths, Bx, T2 = model.logits_bf16(x, mask)
        lp, tok = ops.ctc_frame_topk(logits, Bx, T2, V, lengths, K)
        direct = CTCFusedSearch(lm, Bx, 4, T2, K, DEV, 0.5, 0.2, model.assistor.blank).run(lp, tok, lengths)
        _, _, want, _ = ctc_align_logits(logits, lengths, Bx, T2, V, ids[:, 0, :min(T2, 1023)], n[:, 0], model.assistor.blank)
    assert all(torch.equal(a, b) for a, b in zip(direct, (ids, n, sc)))
    assert torch.equal(spans, want)
    best = rec.recognize(x, mask)
    assert best == [ids[b, 0, :n[b, 0]].tolist() for b in range(2)]
    unfused = CTCRecognizer(model, lm=lm, lm_weight=0.5, beam_width=4, mode='beam')
    ids0, _, sc0 = unfused.recognize_ids(x, mask)
    assert not torch.equal(sc0, sc)
