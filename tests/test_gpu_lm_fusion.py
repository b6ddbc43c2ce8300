"""Shallow fusion on the captured decode step (recognize.BeamDecoder with lm=): the Transformer LM's KV cache (lm.LMCache)
against the full-prefix recompute and the bf16-policy oracle, the fused search in lockstep with the oracle's beam step on
the per-step graph path, graph against eager, the recurrent LM's results unchanged from the host loop that re-read the
prefixes, the decode_step seam with cache['lm'], and recapture after the LM's weights or lm_weight change."""
import pytest
import torch

from tests import ctc_prefix_ref as cpr

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200.lm import RecurrentLanguageModel, TransformerLanguageModel
    from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer, lm_log_probs
    DEV = torch.device('cuda:0')

from oracle import beam_search as obs
from oracle import speech_model as om

REL_L2_LOGITS = 2e-2
V = 4234
LMW = 0.3


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-12))


def _tlm(d=256, H=4, blocks=2, seed=77):
    torch.manual_seed(seed)
    lm = TransformerLanguageModel(dict(type='transformer_lm', vocab_size=V, num_blocks=blocks, d_model=d, n_heads=H,
                                       d_ff=1024, residual_dropout=0.0, smoothing=0.1, share_embedding=True)).eval()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in lm.named_parameters():
            if 'norm' in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n.endswith('.bias'):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    sd = {'lm.' + k: v.detach().clone().float() for k, v in lm.state_dict().items()}
    return lm.to(DEV), sd


def _rnnlm(seed=77):
    torch.manual_seed(seed)
    lm = RecurrentLanguageModel(dict(type='rnn_lm', vocab_size=V, num_layers=2, hidden_size=256, residual_dropout=0.1,
                                     smoothing=0.1, dropout=0.0, share_embedding=True)).eval()
    with torch.no_grad():
        lm.output_project.bias.normal_(0.0, 0.1)
    return lm.to(DEV)


def _lm(kind):
    return _tlm()[0] if kind == 'transformer' else _rnnlm()


def _speech(ctc_weight=0.0, eos_bias=None):
    from tests.test_gpu_model import _build, _params
    params = _params(n_enc=1, n_dec=2)
    if ctc_weight:
        params['ctc_weight'] = ctc_weight
        params['encoder_output_size'] = 256
    model, _ = _build(params)
    with torch.no_grad():
        if ctc_weight:
            model.assistor.output_layer.weight.mul_(8.0)
        if eos_bias is not None:
            model.decoder.output_layer.bias[1] = eos_bias
    return model


def _inputs(B, T, lens, seed=0):
    from tests.test_gpu_model import _batch
    x, mask = _batch(B, T, 80, lens, seed=seed)
    return x.to(DEV), mask.to(DEV)


def _start(B, beam):
    preds = torch.ones(B * beam, 1, dtype=torch.long)
    scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
    return preds, scores, torch.zeros_like(scores, dtype=torch.bool)


# ------------------------------------------------------------------------------------------------ the cache itself
@pytest.mark.parametrize('d,H,max_len,steps,oracle_every', [(256, 4, 14, 12, 1), (192, 2, 14, 12, 1), (256, 4, 300, 300, 23)],
                         ids=['dk64', 'dk96', 'dk64-300-steps'])
def test_cached_lm_matches_the_full_prefix(d, H, max_len, steps, oracle_every):
    """predict(prefix, True, cache) with random parent reorders after every step: the log-probs of each step against predict
    on the explicitly reordered prefix (the reference's recompute) and against the bf16-policy oracle."""
    lm, sd = _tlm(d, H)
    N = 6
    g = torch.Generator().manual_seed(5)
    prefix = torch.ones(N, 1, dtype=torch.long)
    worst_full = worst_ref = 0.0
    with torch.no_grad():
        cache = lm.init_cache(N, max_len)
        for s in range(steps):
            got = lm.predict(prefix.to(DEV), True, cache)
            assert got.shape == (N, 1, V) and cache.step == s + 1
            full = lm.predict(prefix.to(DEV), last_frame=True)
            worst_full = max(worst_full, _rel(got, full))
            if s % oracle_every == 0 or s == steps - 1:
                ref = om.transformer_lm_log_probs(prefix, sd, 'lm.', 2, H, last_frame=True, policy='bf16')
                worst_ref = max(worst_ref, _rel(got, ref))
            parent = torch.randint(0, N, (N,), generator=g)
            tok = torch.randint(2, V, (N, 1), generator=g)
            cache.reorder(parent.to(DEV))
            prefix = torch.cat((prefix[parent], tok), dim=1)
    print(f'd_k {d // H}, {steps} steps: cached vs full prefix rel_l2<={worst_full:.3e}, vs oracle rel_l2<={worst_ref:.3e}')
    assert worst_full < REL_L2_LOGITS and worst_ref < REL_L2_LOGITS


# ------------------------------------------------------------------------------------------------ the fused search
@pytest.mark.parametrize('ctc_weight', [0.0, 0.3])
@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_fused_search_lockstep_on_the_graph_path(kind, ctc_weight):
    """The captured step with the LM inside it, replayed step by step (keep_logp=True keeps the fused log-probs): the
    oracle's beam_step fed those log-probs makes the same choices with the same score bits and flags at every step, and
    finalize equals beam_finalize; with the CTC term the float64 restatement of joint decoding (JointSearch) is fed the
    attention and LM log-probs.  The LM's log-probs inside the step equal lm_log_probs on the reconstructed prefixes: bit
    for bit for the recurrent LM, within REL_L2_LOGITS for the cached Transformer LM."""
    model = _speech(ctc_weight)
    lm = _lm(kind)
    B, beam, max_len, P = 2, 3, 8, 6
    x, mask = _inputs(B, 160, [160, 131], seed=6)
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x, mask)
        ctc = (model.assistor, ctc_weight, P) if ctc_weight else None
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=True, keep_logp=True, ctc=ctc, lm=(lm, LMW))
        assert not bd.persistent
        bd.setup(mem, lens)
        preds, scores, flag = _start(B, beam)
        js = cpr.JointSearch(bd.ctc.lp.view(B, T2, V).cpu(), lens.cpu().tolist(), beam, P, ctc_weight, LMW) if ctc else None
        worst = 0.0
        for s in range(max_len):
            prefix = bd.state.reconstruct(s)
            bd.step()
            assert bd.graph is not None
            lm_cpu = bd.lm_logp.cpu()
            want = lm_log_probs(lm, prefix).cpu()
            if kind == 'rnn':
                assert torch.equal(lm_cpu, want), f'recurrent LM log-probs differ at step {s}'
            else:
                worst = max(worst, _rel(lm_cpu, want))
            fused = bd.logp.cpu()
            if ctc is None:
                preds, scores, flag = obs.beam_step(fused, preds, scores, flag, beam)
                assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'ids differ at step {s}'
                assert torch.equal(bd.state.scores.cpu().view(torch.int32), scores.view(-1).view(torch.int32)), s
                assert torch.equal(bd.state.flag.cpu().bool(), flag.view(-1)), s
            else:
                js.step(fused.double() - LMW * lm_cpu.double(), lm_cpu)
                assert torch.equal(bd.state.reconstruct(s + 1).cpu(), js.preds), f'prefixes differ at step {s}'
                got, ref = bd.state.scores.cpu().double(), js.scores.view(-1)
                assert torch.equal(torch.isfinite(got), torch.isfinite(ref)), s
                assert float((got - ref)[torch.isfinite(ref)].abs().max()) < 1e-3, s
        if ctc is None:
            nb, ns = obs.beam_finalize(preds, scores, beam, 2, 0.6, 5)
            gp, gs = bd.state.finalize(0.6, 5, 2)
            assert torch.equal(gp[:, :, :max_len].cpu(), nb)
            assert torch.equal(gs.cpu(), ns)
    print(f'{kind} LM, ctc_weight {ctc_weight}: LM log-probs in the step vs lm_log_probs rel_l2<={worst:.3e}')
    assert worst < REL_L2_LOGITS


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_graph_equals_eager_and_natural_end(kind):
    """recognize_ids on the graph and the eager path: the same ids, score bits and executed steps, with and without the
    CTC term.  With a decoder that ends early, the graph path stops at the step the oracle loop ends at, and the replays a
    polling host launches after the end leave the search state untouched."""
    lm = _lm(kind)
    B, beam, max_len = 3, 4, 10
    x, mask = _inputs(B, 200, [200, 150, 173])
    for ctc_weight in (0.0, 0.3):
        model = _speech(ctc_weight)
        kw = dict(lm=lm, lm_weight=LMW, ctc_weight=ctc_weight, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6,
                  lamda=5, ngpu=1)
        rec_g, rec_e = SpeechToTextRecognizer(model, **kw), SpeechToTextRecognizer(model, use_graph=False, **kw)
        p1, s1, n1 = rec_e.recognize_ids(x, mask)
        p2, s2, n2 = rec_g.recognize_ids(x, mask)
        p3, s3, n3 = rec_g.recognize_ids(x, mask)            # the second call replays the captured step
        bd = next(iter(rec_g._decoders.values()))
        assert bd.use_graph and bd.graph is not None and not bd.persistent and bd.lm is lm
        assert n1 == n2 == n3 == max_len
        assert torch.equal(p1, p2) and torch.equal(p2, p3)
        assert torch.equal(s1.view(torch.int32), s2.view(torch.int32)) and torch.equal(s2, s3)
    # natural end: the decoder's <S/E> bias makes every hypothesis end within a few steps
    model = _speech(eos_bias=1e4)
    max_len = 20
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x, mask)
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False, lm=(lm, LMW))
        bd.setup(mem, lens)
        preds, scores, flag = _start(B, beam)
        end = None
        for s in range(max_len):
            bd.step()
            preds, scores, flag = obs.beam_step(bd.logp.cpu(), preds, scores, flag, beam)
            if bool(flag.all()):
                end = s + 1
                break
    assert end is not None and end < 8, end                   # ends before the first poll (every 8 steps)
    rec = SpeechToTextRecognizer(model, lm=lm, lm_weight=LMW, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6,
                                 lamda=5, ngpu=1)
    ids, sc, n = rec.recognize_ids(x, mask)
    assert n == end
    bd = next(iter(rec._decoders.values()))
    st = bd.state
    before = [t.clone() for t in (st.tok_hist, st.par_hist, st.last_tok, st.scores, st.flag, st.anc, st.ctrl)]
    with torch.no_grad():
        for _ in range(3):
            bd.step()
    torch.cuda.synchronize()
    for t, b in zip((st.tok_hist, st.par_hist, st.last_tok, st.scores, st.flag, st.anc, st.ctrl), before):
        assert torch.equal(t, b)


def _old_fused_loop(model, lm, x, mask, B, beam, max_len):
    """The search as it ran before the LM entered the captured step: lm_log_probs on the reconstructed prefixes, then the
    eager step of an LM-less BeamDecoder, polling the end after every step."""
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x, mask)
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False)
        bd.setup(mem, lens)
        bd.lm_weight = LMW
        for i in range(max_len):
            bd.lm_logp = lm_log_probs(lm, bd.state.reconstruct(i))
            bd._step_kernels()
            if int(bd._read_ctrl()[1]):
                break
        steps = int(bd._read_ctrl()[0])
        preds, scores = bd.state.finalize(0.6, 5, 2)
    return preds[:, :, :steps], scores, steps


@pytest.mark.parametrize('eos_bias', [None, 1e4])
def test_rnn_lm_results_unchanged(eos_bias):
    """The recurrent LM reads the newest token from a zero state either way, so recognize_ids returns exactly what the host
    loop returned: the same ids, the same score bits and the same step count."""
    lm = _rnnlm()
    model = _speech(eos_bias=eos_bias)
    B, beam, max_len = 3, 4, 12
    x, mask = _inputs(B, 200, [200, 150, 173])
    p0, s0, n0 = _old_fused_loop(model, lm, x, mask, B, beam, max_len)
    rec = SpeechToTextRecognizer(model, lm=lm, lm_weight=LMW, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6,
                                 lamda=5, ngpu=1)
    p1, s1, n1 = rec.recognize_ids(x, mask)
    assert n1 == n0 and torch.equal(p1, p0) and torch.equal(s1.view(torch.int32), s0.view(torch.int32))


# ------------------------------------------------------------------------------------------------ the seam
def test_lm_cache_through_the_decode_step_seam():
    """decode_step with cache = {'decoder': DecoderCache, 'lm': LMCache} (the reorder the reference left commented out,
    speech2text.py:142-143) against the same loop with cache['lm'] None (the full-prefix LM, the reference's behaviour),
    a lockstep run in which the oracle's beam_step drives both reorders, and the cache's refusals."""
    lm, sd = _tlm()
    model = _speech()
    B, beam, max_len = 3, 4, 8
    N = B * beam
    x, mask = _inputs(B, 200, [200, 150, 173])
    rec = SpeechToTextRecognizer(model, lm=lm, lm_weight=LMW, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6,
                                 lamda=5, ngpu=1)
    memory, mmask, _, _ = rec.encode(x, mask)
    T2 = memory.shape[1]
    bm = memory.unsqueeze(1).repeat(1, beam, 1, 1).view(N, T2, -1)
    bmask = mmask.unsqueeze(1).repeat(1, beam, 1).view(N, T2)

    def loop(cache):
        preds, scores, flag = (t.to(DEV) for t in _start(B, beam))
        with torch.no_grad():
            for _ in range(max_len):
                preds, cache, scores, flag = rec.decode_step(preds, bm, bmask, cache, scores, flag)
        return preds, scores

    with torch.no_grad():
        dc, lc = model.decoder.init_cache(bm, bmask, max_len, beam=beam), lm.init_cache(N, max_len)
    p_c, s_c = loop({'decoder': dc, 'lm': lc})
    with torch.no_grad():
        dc2 = model.decoder.init_cache(bm, bmask, max_len, beam=beam)
    p_f, s_f = loop({'decoder': dc2, 'lm': None})
    assert lc.step == max_len
    same = int((p_c == p_f).all(dim=1).sum())
    print(f'LM-cached seam vs full-prefix seam: {same}/{N} hypotheses identical')
    torch.testing.assert_close(s_c, s_f, rtol=3e-2, atol=0.3)
    assert torch.equal(p_c.view(B, beam, -1)[:, 0], p_f.view(B, beam, -1)[:, 0]), '1-best of the cached and the recomputing seam differ'
    # lockstep: the oracle's beam_step picks the parents and both caches follow them
    with torch.no_grad():
        dc, lc = model.decoder.init_cache(bm, bmask, max_len, beam=beam), lm.init_cache(N, max_len)
        o_preds, o_scores, o_flag = _start(B, beam)
        for s in range(max_len):
            preds = o_preds.to(DEV)
            lp, dc, _ = model.decoder.inference(preds, bm, bmask, dc)
            lm_lp = lm.predict(preds, True, lc).squeeze(1)
            ref = om.transformer_lm_log_probs(o_preds, sd, 'lm.', 2, 4, last_frame=True, policy='bf16').squeeze(1)
            alive = ~o_flag.view(-1)
            assert _rel(lm_lp.cpu()[alive], ref[alive]) < REL_L2_LOGITS, s
            tr = []
            o_preds, o_scores, o_flag = obs.beam_step(lp.cpu(), o_preds, o_scores, o_flag, beam, lm_log_probs=lm_lp.cpu(),
                                                      lm_weight=LMW, trace=tr)
            dc.reorder(tr[0]['parent'].to(DEV))
            lc.reorder(tr[0]['parent'].to(DEV))
    assert torch.equal(o_preds, p_c.cpu()), 'lockstep ids differ from the seam'
    # misuse
    with torch.no_grad():
        lc = lm.init_cache(N, 2)
        one = torch.ones(N, 1, dtype=torch.long, device=DEV)
        with pytest.raises(RuntimeError, match='reorder before the first inference step'):
            lc.reorder(torch.arange(N, device=DEV))
        with pytest.raises(ValueError, match='one new token per call'):
            lm.predict(torch.ones(N, 2, dtype=torch.long, device=DEV), True, lc)
        with pytest.raises(ValueError, match='last_frame must be True'):
            lm.predict(one, False, lc)
        lm.predict(one, True, lc)
        lc.advance_without_reorder()
        lm.predict(torch.ones(N, 2, dtype=torch.long, device=DEV), True, lc)
        lc.advance_without_reorder()
        with pytest.raises(ValueError, match='LMCache is full'):
            lm.predict(torch.ones(N, 3, dtype=torch.long, device=DEV), True, lc)
        lc = lm.init_cache(N, 4)
        lm.load_state_dict(_tlm(seed=78)[0].state_dict())
        with pytest.raises(RuntimeError, match='different LM weights'):
            lm.predict(one, True, lc)


# ------------------------------------------------------------------------------------------------ weights move
@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_recapture_after_the_lm_or_its_weight_changes(kind):
    """The captured step bakes in the LM's packed weights and lm_weight: after lm.load_state_dict or a new rec.lm_weight
    the next recognize_ids equals a freshly built recognizer's."""
    model = _speech()
    lm = _lm(kind)
    other = (_tlm(seed=78)[0] if kind == 'transformer' else _rnnlm(seed=78)).state_dict()
    B, beam, max_len = 2, 3, 6
    x, mask = _inputs(B, 160, [160, 131])
    kw = dict(beam_width=beam, nbest=2, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    rec = SpeechToTextRecognizer(model, lm=lm, lm_weight=LMW, **kw)
    p0, s0, _ = rec.recognize_ids(x, mask)
    lm.load_state_dict(other)
    p1, s1, _ = rec.recognize_ids(x, mask)
    q1, t1, _ = SpeechToTextRecognizer(model, lm=lm, lm_weight=LMW, **kw).recognize_ids(x, mask)
    assert torch.equal(p1, q1) and torch.equal(s1, t1)
    assert not torch.equal(s0, s1)
    rec.lm_weight = 0.7
    p2, s2, _ = rec.recognize_ids(x, mask)
    q2, t2, _ = SpeechToTextRecognizer(model, lm=lm, lm_weight=0.7, **kw).recognize_ids(x, mask)
    assert torch.equal(p2, q2) and torch.equal(s2, t2)
    assert not torch.equal(s1, s2)
