"""GPU checks of n-best rescoring (DESIGN.md 4.10): otb_token_logprob against float64, otb_nbest_rescore against the
restatement (tests/rescore_ref.py) on the kernel's own token log-probs, TransformerDecoder.score_bf16 against forward_bf16,
and the recognizers end to end against the restatement run on their own first-pass n-best."""
import pytest
import torch

from oracle import speech_model as om
from tests import rescore_ref as rr

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    from opentransformer_b200.recognize import CTCRecognizer, SpeechToTextRecognizer, ctc_decode
    DEV = torch.device('cuda:0')

EOS, NEG_INF = rr.EOS, rr.NEG_INF


# ------------------------------------------------------------------------------------------------ otb_token_logprob
@pytest.mark.parametrize('V', [40, 4234])
@pytest.mark.parametrize('rows', [1, 333, 20000])
def test_token_logprob_matches_float64(V, rows):
    """Padded row pitch, mixed -1 targets, rows of logits at +-1e4; |error| <= 2e-5 max(1, |value|) (at |logit| 1e4 an fp32
    ulp is 1e-3, so the bound is relative there); a second call is bit-identical."""
    g = torch.Generator().manual_seed(rows + V)
    ld = (V + 7) // 8 * 8 + (64 if rows % 2 else 0)
    logits = torch.full((rows, ld), float('nan'))                  # pad columns must not be read
    logits[:, :V] = 4.0 * torch.randn(rows, V, generator=g)
    big = torch.rand(rows, generator=g) < 0.1
    logits[big, :V] = 1e4 * (2 * torch.rand(int(big.sum()), V, generator=g) - 1)
    target = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32)
    target[torch.rand(rows, generator=g) < 0.2] = -1
    x, t = logits.to(DEV), target.to(DEV)
    got = ops.token_logprob(x, V, t)
    ref = torch.log_softmax(x[:, :V].double(), dim=-1).gather(1, t.long().clamp_min(0)[:, None])[:, 0]
    ref = torch.where(t >= 0, ref, torch.zeros_like(ref))
    err = ((got.double() - ref).abs() / ref.abs().clamp_min(1.0)).max()
    assert float(err) <= 2e-5, float(err)
    assert bool((got[t < 0] == 0).all())
    assert torch.equal(ops.token_logprob(x, V, t), got)


def test_token_logprob_refuses_unaligned_rows():
    x = torch.zeros(4, 42, device=DEV)
    with pytest.raises(RuntimeError, match='16-byte aligned'):
        ops.token_logprob(x, 40, torch.zeros(4, dtype=torch.int32, device=DEV))


# ------------------------------------------------------------------------------------------------ otb_nbest_rescore
def _first_pass(B, K, Lp, V, g):
    """Random cut hypotheses with planted duplicates: -> (hyps [B][K] lists, tgt i32 [B, K, Lp], n i32 [B, K])."""
    hyps = []
    for b in range(B):
        row = []
        for k in range(K):
            if k > 0 and torch.rand(1, generator=g) < 0.3:
                row.append(list(row[int(torch.randint(0, k, (1,), generator=g))]))
            else:
                row.append(torch.randint(2, V, (int(torch.randint(0, Lp, (1,), generator=g)),), generator=g).tolist())
        hyps.append(row)
    tgt = torch.full((B, K, Lp), -1, dtype=torch.int32)
    for b in range(B):
        for k in range(K):
            y = hyps[b][k] + [EOS]
            tgt[b, k, :len(y)] = torch.tensor(y, dtype=torch.int32)
    n = torch.tensor([[len(y) for y in row] for row in hyps], dtype=torch.int32)
    return hyps, tgt, n


@pytest.mark.parametrize('K,M,weight,ties', [(1, 1, 1.0, False), (5, 1, 0.7, False), (16, 2, 0.3, False), (16, 2, 1.0, True),
                                             (12, 1, 0.0, False)])
def test_nbest_rescore_matches_the_restatement(K, M, weight, ties):
    """The kernel's own token log-probs through the restatement's float32 sums: identical ids, lengths, order and scores.
    ties: log-probs and first-pass scores on a 1/8 grid, so many hypotheses tie exactly and the first-pass order decides."""
    B, Lp, V, width = 9, 14, 50, 13
    g = torch.Generator().manual_seed(K * 10 + M)
    hyps, tgt, n = _first_pass(B, K, Lp, V, g)
    if ties:
        tok = torch.zeros(M, B, K, Lp)
        tok[tgt.expand(M, -1, -1, -1) >= 0] = -torch.randint(0, 3, (int((tgt >= 0).sum()) * M,), generator=g).float() / 8
        s1 = -torch.randint(0, 3, (B, K), generator=g).float() / 8
    else:
        logits = 3.0 * torch.randn(M * B * K * Lp, (V + 7) // 8 * 8, generator=g)
        tok = ops.token_logprob(logits.to(DEV), V, tgt.repeat(M, 1, 1).view(-1).to(DEV)).view(M, B, K, Lp).cpu()
        s1 = torch.sort(-5.0 * torch.rand(B, K, generator=g), dim=1, descending=True).values
    nbest = max(1, K - 2)
    ids, lens, sc = ops.nbest_rescore(tgt.to(DEV), n.to(DEV), s1.to(DEV), tok.to(DEV), weight, nbest, width, EOS)
    for b in range(B):
        tl = [[tok[m, b, k, :n[b, k] + 1] for m in range(M)] for k in range(K)]
        ranked = rr.rerank(hyps[b], s1[b].tolist(), tl, weight, nbest, dtype=torch.float32)
        want_ids, want_len, want_sc = rr.as_tensors(ranked, width)
        assert torch.equal(ids[b].cpu(), want_ids), b
        assert lens[b].tolist() == want_len.tolist(), b
        assert torch.equal(sc[b].cpu(), want_sc.float()), b
    if ties:
        assert len({float(v) for v in sc[sc > NEG_INF].cpu()}) < int((sc > NEG_INF).sum())     # ties did occur


# ------------------------------------------------------------------------------------------------ score_bf16
def _speech_model(ctc_weight=0.0, n_dec=2, eos_bias=-1e4):
    from tests.test_gpu_model import _build, _params
    params = _params(n_enc=1, n_dec=n_dec)
    params['ctc_weight'] = ctc_weight
    params['encoder_output_size'] = 256
    model, sd = _build(params)
    with torch.no_grad():
        if ctc_weight > 0.0:
            model.assistor.output_layer.weight.mul_(8.0)
            for k, v in model.assistor.state_dict().items():
                sd[f'assistor.{k}'] = v.detach().clone().float().cpu()
        model.decoder.output_layer.bias[1] = eos_bias
        sd['decoder.output_layer.bias'] = model.decoder.output_layer.bias.detach().clone().float().cpu()
    return model, sd, params


def _inputs(B, T, lens, seed=0):
    from tests.test_gpu_model import _batch
    x, mask = _batch(B, T, 80, lens, seed=seed)
    return x.to(DEV), mask.to(DEV)


def test_score_bf16_matches_forward_bf16_on_tiled_memory():
    from tests.test_gpu_model import MAX_ABS_FRAC, REL_L2_LOGITS, _rel
    model, _, _ = _speech_model()
    B, K, Lp = 3, 5, 11
    x, mask = _inputs(B, 200, [200, 150, 97])
    with torch.no_grad():
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
        g = torch.Generator().manual_seed(5)
        inputs = torch.randint(2, model.decoder.vocab_size, (B * K, Lp), generator=g).to(DEV)
        got = model.decoder.score_bf16(inputs, mem, mem_len, B, K, Lp, T2)
        tiled = mem.view(B, 1, T2, -1).expand(B, K, T2, mem.shape[1]).reshape(B * K * T2, -1).contiguous()
        want = model.decoder.forward_bf16(inputs, tiled, mem_len.repeat_interleave(K), B * K, Lp, T2)
    V = model.decoder.vocab_size
    got, want = got[:, :V], want[:, :V]
    identical = torch.equal(got, want)
    print(f'score_bf16 vs forward_bf16 on tiled memory: bit-identical = {identical}')
    assert _rel(got, want) <= REL_L2_LOGITS
    assert float((got - want).abs().max()) <= MAX_ABS_FRAC * float(want.abs().max())


# ------------------------------------------------------------------------------------------------ end to end
def _tol(s):
    return 0.3 + 3e-2 * abs(s)                  # the bf16-policy tolerance of the beam-search scores (test_gpu_model)


def _check_against_restatement(ids, lens, scores, hyps, s1, second, weight, nbest):
    """Per utterance: the port's rescored n-best (ids, lens, scores) against the restatement on the same first-pass
    hypotheses `hyps` (cut) and scores s1, with second(b, y) -> the float64 token log-probs of each second-pass model."""
    for b in range(len(hyps)):
        tl = [second(b, y) for y in hyps[b]]
        ref = rr.rerank(hyps[b], s1[b], tl, weight, len(hyps[b]))
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


def _decoder_second(model, sd, params, mem, mem_len, T2):
    memory = mem.float().view(-1, T2, mem.shape[1]).cpu()
    kw = om.decoder_kwargs(params)
    return lambda b, y: rr.decoder_token_logprobs(y, memory[b], int(mem_len[b]), sd, 'decoder.', policy='bf16', **kw)


def _transformer_lm(V):
    from opentransformer_b200.lm import TransformerLanguageModel
    torch.manual_seed(11)
    p = dict(type='transformer_lm', vocab_size=V, num_blocks=2, d_model=256, n_heads=4, d_ff=1024, residual_dropout=0.0,
             smoothing=0.1, share_embedding=True)
    lm = TransformerLanguageModel(p)
    with torch.no_grad():
        lm.embedding.weight.mul_(0.05)
        lm.output_project.bias.normal_(0.0, 0.5)
    sd = {k: v.detach().clone().float() for k, v in lm.state_dict().items()}
    return lm.to(DEV), lambda b, y: rr.transformer_lm_token_logprobs(y, sd, '', 2, 4, policy='bf16')


def _rnn_lm(V):
    from tests.test_gpu_rnnlm import _lm
    lm, sd, _ = _lm(64, V=V)
    return lm, lambda b, y: rr.rnn_lm_token_logprobs(y, sd, '', 2, policy='bf16')


@pytest.mark.parametrize('with_lm', [None, 'transformer'])
def test_attention_rescoring_of_the_ctc_nbest(with_lm):
    """apply_rescoring (and with an LM, both second-pass terms): the CTC prefix beam search's n-best of the joint-CTC head,
    re-ranked by the attention decoder."""
    model, sd, params = _speech_model(ctc_weight=0.3, eos_bias=0.0)
    B, beam, nbest, w = 3, 6, 4, 0.7
    V = model.decoder.vocab_size
    x, mask = _inputs(B, 240, [240, 200, 131], seed=2)
    lm, lm_second = _transformer_lm(V) if with_lm else (None, None)
    rec = SpeechToTextRecognizer(model, lm=lm, beam_width=beam, nbest=nbest, apply_rescoring=True,
                                 apply_lm_rescoring=lm is not None, rescore_weight=w)
    ids, scores, steps = rec.recognize_ids(x, mask)
    assert not rec._decoders                                   # no attention beam search ran
    with torch.no_grad():
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
        cids, cn, csc = ctc_decode(model.assistor.logits_bf16(mem), mem_len, B, T2, V, 0, 'beam', beam)
    hyps = [[rr.cut(cids[b, k].tolist(), int(cn[b, k])) for k in range(beam)] for b in range(B)]
    assert ids.shape == (B, nbest, steps) and steps == max(len(y) for row in hyps for y in row) + 1
    lens = (ids == EOS).int().argmax(dim=2)
    dec = _decoder_second(model, sd, params, mem, mem_len, T2)
    second = (lambda b, y: [dec(b, y), lm_second(b, y)]) if lm is not None else (lambda b, y: [dec(b, y)])
    _check_against_restatement(ids.cpu(), lens.cpu(), scores.cpu(), hyps, csc.cpu().tolist(), second, w, nbest)


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_lm_rescoring_keeps_the_persistent_first_pass(kind):
    """apply_lm_rescoring: the search runs on the persistent kernel without the LM, its beam_width-best equal bit for bit
    to recognize_ids of a recognizer without an LM; then the LM re-ranks them."""
    model, _, _ = _speech_model(eos_bias=0.0)
    B, beam, nbest, w, L = 4, 5, 3, 0.5, 16
    V = model.decoder.vocab_size
    x, mask = _inputs(B, 400, [400, 377, 250, 181], seed=4)
    lm, lm_second = _transformer_lm(V) if kind == 'transformer' else _rnn_lm(V)
    kw = dict(beam_width=beam, max_len=L, penalty=0.6, lamda=5)
    rec = SpeechToTextRecognizer(model, lm=lm, nbest=nbest, apply_lm_rescoring=True, rescore_weight=w, **kw)
    ids, scores, steps = rec.recognize_ids(x, mask)
    bd = next(iter(rec._decoders.values()))
    assert bd.persistent
    first, first_sc = bd.state.finalize(0.6, 5, beam)          # the search state the rescoring started from
    p0, s0, n0 = SpeechToTextRecognizer(model, nbest=beam, **kw).recognize_ids(x, mask)
    assert n0 == steps and torch.equal(first[:, :, :steps], p0) and torch.equal(first_sc, s0)
    hyps = [[rr.cut(p0[b, k].tolist()) for k in range(beam)] for b in range(B)]
    assert ids.shape == (B, nbest, steps)
    lens = (torch.cat((ids, torch.full((B, nbest, 1), EOS, device=DEV)), 2) == EOS).int().argmax(dim=2)
    _check_against_restatement(ids.cpu(), lens.cpu(), scores.cpu(), hyps, s0.cpu().tolist(), lambda b, y: [lm_second(b, y)], w,
                               nbest)


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_ctc_recognizer_lm_rescoring(kind):
    from tests.test_gpu_ctc_model import _build, _params
    model, _ = _build(_params('transformer', V=40))
    B, beam, w = 3, 8, 1.0
    x, mask = _inputs(B, 200, [200, 160, 181], seed=1)
    lm, lm_second = _transformer_lm(40) if kind == 'transformer' else _rnn_lm(40)
    rec = CTCRecognizer(model, lm=lm, beam_width=beam, mode='beam', apply_lm_rescoring=True, rescore_weight=w)
    ids, lens, scores = rec.recognize_ids(x, mask)
    cids, cn, csc = CTCRecognizer(model, beam_width=beam, mode='beam').recognize_ids(x, mask)
    assert ids.shape == cids.shape
    assert bool((ids.cpu() * (torch.arange(ids.shape[2]) >= lens.cpu()[..., None]) == 0).all())    # 0 after the end
    hyps = [[rr.cut(cids[b, k].tolist(), int(cn[b, k])) for k in range(beam)] for b in range(B)]
    _check_against_restatement(ids.cpu(), lens.cpu(), scores.cpu(), hyps, csc.cpu().tolist(), lambda b, y: [lm_second(b, y)], w,
                               beam)
    spans = rec.recognize_spans(x, mask)[3]
    assert spans.shape[1] == ids.shape[2] and torch.equal(rec.recognize_spans(x, mask)[0], ids)


def test_recognize_spans_aligns_the_rescored_best():
    from opentransformer_b200.model import ctc_align_logits
    model, _, _ = _speech_model(ctc_weight=0.3, eos_bias=0.0)
    B = 3
    x, mask = _inputs(B, 240, [240, 200, 131], seed=2)
    rec = SpeechToTextRecognizer(model, beam_width=6, nbest=2, apply_rescoring=True, rescore_weight=0.7)
    ids, scores, steps, spans = rec.recognize_spans(x, mask)
    ids2, scores2, steps2 = rec.recognize_ids(x, mask)
    assert steps == steps2 and torch.equal(ids, ids2) and torch.equal(scores, scores2)
    with torch.no_grad():
        mem, mem_len, _, T2 = model.encode_bf16(x, mask)
        best = torch.cat((ids[:, 0], torch.full((B, 1), EOS, dtype=ids.dtype, device=DEV)), dim=1)
        n_tok = (best == EOS).int().argmax(dim=1) + 1
        want = ctc_align_logits(model.assistor.logits_bf16(mem), mem_len, B, T2, model.decoder.vocab_size, best, n_tok, 0)[2]
    assert torch.equal(spans, want)
