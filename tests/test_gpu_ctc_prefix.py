"""GPU checks of joint CTC/attention decoding: the CTC prefix kernels (csrc/ctc_prefix.cu) against the float64 restatement
(tests/ctc_prefix_ref.py), the search with the CTC term in lockstep with the restatement, graph against eager, a case where
the CTC term has to change the answer, ctc_weight 0 leaving today's path alone, and recognize_spans."""
import pytest
import torch

from tests import ctc_prefix_ref as cpr

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer, lm_log_probs
    DEV = torch.device('cuda:0')

EOS = cpr.EOS
NEG_INF = float('-inf')


def _close(got, want, what, tol=1e-4):
    """got f32 against want f64: the same -inf pattern, no NaN, finite entries within tol (+ 1e-6 relative)."""
    got, want = got.detach().cpu().double(), want.double()
    assert not bool(torch.isnan(got).any()), what
    assert torch.equal(torch.isneginf(got), torch.isneginf(want)), what
    fin = torch.isfinite(want)
    if bool(fin.any()):
        err = (got[fin] - want[fin]).abs() - 1e-6 * want[fin].abs()
        assert float(err.max()) <= tol, (what, float(err.max()))


def _joint_model(n_enc=1, n_dec=2, eos_bias=None):
    from tests.test_gpu_model import _build, _params
    params = _params(n_enc=n_enc, n_dec=n_dec)
    params['ctc_weight'] = 0.3
    params['encoder_output_size'] = 256
    model, _ = _build(params)
    with torch.no_grad():
        model.assistor.output_layer.weight.mul_(8.0)        # a head with opinions: frames that prefer some tokens
        if eos_bias is not None:
            model.decoder.output_layer.bias[1] = eos_bias
    return model


def _inputs(B, T, lens, seed=0):
    from tests.test_gpu_model import _batch
    x, mask = _batch(B, T, 80, lens, seed=seed)
    return x.to(DEV), mask.to(DEV)


# ------------------------------------------------------------------------------------------------ kernels vs restatement
def test_score_and_advance_match_the_restatement():
    """init -> (score -> advance) x 4 on random log-probs with ragged lengths (one utterance of 1 frame, one of 2: shorter
    than the prefixes), survivors picked by hand: two children of one parent, a row that takes <S/E>, a finished row;
    candidates that repeat the last token, name <S/E> and the blank."""
    B, beam, T, V, P, w, lmw, Lmax = 4, 3, 24, 20, 6, 0.3, 0.2, 8
    lens = [24, 1, 2, 17]
    N = B * beam
    g = torch.Generator().manual_seed(0)
    lp = torch.log_softmax(2.0 * torch.randn(B, T, V, generator=g), dim=-1)
    in_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ctc = ops.CTCPrefixState(B, beam, T, V, P, DEV)
    ctc.lp.copy_(lp.view(B * T, V))
    st = ops.BeamState(B, beam, Lmax, DEV)
    st.init()
    ctc.init(in_len)
    state = [cpr.empty_prefix(lp[n // beam], lens[n // beam]) for n in range(N)]
    for n in range(N):
        _close(ctc.gamma[0, n, :lens[n // beam]], state[n][0], f'init gamma {n}')
    assert bool((ctc.psi[0] == 0).all())
    out_val = torch.zeros(N, beam, device=DEV)
    out_idx = torch.zeros(N, beam, dtype=torch.int32, device=DEV)
    last, fin = [EOS] * N, [False] * N
    # per step and utterance-local row: (local parent, candidate slot, or -1 for <S/E>)
    plan = [[(0, 2), (0, 0), (1, 3)], [(0, 0), (0, 1), (2, -1)], [(1, 0), (1, 4), (2, -1)], [(0, 0), (2, -1), (1, 2)]]
    for step in range(4):
        ids = torch.zeros(N, P, dtype=torch.int64)
        for n in range(N):
            first = [last[n]] if step > 0 and not fin[n] else []                  # a candidate that repeats the last token
            first += [EOS] if n % 2 == 0 and EOS not in first else []
            pool = [v for v in (torch.randperm(V - 2, generator=g) + 2).tolist() if v not in first]
            ids[n] = torch.tensor((first + pool)[:P])
        if step == 2:
            ids[0, P - 1] = 0                                                        # the blank among the candidates
        att = -5.0 * torch.rand(N, P, generator=g)
        lm = torch.log_softmax(torch.randn(N, V, generator=g), dim=-1)
        ctc.cand_val.copy_(att + lmw * lm.gather(1, ids))
        ctc.cand_id.copy_(ids.int())
        out_val.fill_(123.0)
        ctc.score(st, in_len, w, out_val, out_idx, lm.to(DEV), lmw)
        cand_state = [None] * N
        for n in range(N):
            if fin[n]:
                assert bool((out_val[n] == 123.0).all())                             # finished rows are left to the beam step
                continue
            u = n // beam
            gam, psi = cpr.extend(lp[u], lens[u], state[n][0], step == 0, last[n], ids[n])
            cand_state[n] = (gam, psi)
            _close(ctc.gamma_cand[n, :, :lens[u]], gam, f'gamma_cand step {step} row {n}')
            _close(ctc.psi_cand[n], psi, f'psi_cand step {step} row {n}')
            d = torch.where(torch.isneginf(psi), psi, psi - state[n][1])
            lmv = lmw * lm[n, ids[n]].double()
            joint = torch.where(torch.isneginf(d), d, (1 - w) * att[n].double() + w * d + lmv)
            order = sorted(range(P), key=lambda j: (-float(joint[j]), int(ids[n, j])))
            want = joint[order[:beam]]
            _close(out_val[n], want, f'joint step {step} row {n}')
            margin = float((joint[order[:beam]] - joint[order[1:beam + 1]]).nan_to_num(nan=0.0).min())
            if margin > 1e-3 or bool(torch.isneginf(joint).all()):                   # all -inf: ties go to the lower id
                assert out_idx[n].tolist() == [int(ids[n, j]) for j in order[:beam]], (step, n)
        # ---- survivors written by hand, as the beam step would leave them
        par = torch.zeros(N, dtype=torch.int32)
        tok = torch.zeros(N, dtype=torch.int32)
        for u in range(B):
            for r, (pl, slot) in enumerate(plan[step]):
                p = u * beam + pl
                par[u * beam + r] = p
                tok[u * beam + r] = EOS if slot < 0 or fin[p] else int(ids[p, slot])
        st.par_hist[step].copy_(par)
        st.tok_hist[step].copy_(tok)
        st.last_tok.copy_(tok.long())
        st.flag.copy_((tok == EOS).to(torch.uint8))
        st.ctrl[0] = step + 1
        ctc.advance(st, in_len)
        new_state, nxt = [], (step + 1) & 1
        for nn in range(N):
            p, c = int(par[nn]), int(tok[nn])
            if c == EOS:
                new_state.append(state[p])
            else:
                j = ids[p].tolist().index(c)
                new_state.append((cand_state[p][0][j], cand_state[p][1][j]))
            _close(ctc.gamma[nxt, nn, :lens[nn // beam]], new_state[-1][0], f'advance gamma step {step} row {nn}')
            _close(ctc.psi[nxt, nn], new_state[-1][1], f'advance psi step {step} row {nn}')
        state, last, fin = new_state, tok.tolist(), (tok == EOS).tolist()
    # once the search has ended, score and advance leave everything alone
    st.ctrl[1] = 1
    before = (ctc.gamma.clone(), ctc.psi_cand.clone())
    out_val.fill_(7.0)
    ctc.score(st, in_len, w, out_val, out_idx)
    ctc.advance(st, in_len)
    assert torch.equal(before[0], ctc.gamma) and torch.equal(before[1], ctc.psi_cand) and bool((out_val == 7.0).all())


def test_complete_hypothesis_scores_as_the_ctc_loss():
    """psi of <S/E> after a hypothesis = -nll of otb_ctc_loss for the hypothesis plus <S/E>, through score / advance."""
    B, beam, T, V, P = 3, 1, 40, 30, 4
    lens = [40, 25, 9]
    g = torch.Generator().manual_seed(3)
    logits = (2.0 * torch.randn(B * T, (V + 7) // 8 * 8, generator=g)).to(DEV)
    y = torch.randint(2, V, (B, 5), generator=g)
    y[:, 2] = y[:, 1]
    in_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ctc = ops.CTCPrefixState(B, beam, T, V, P, DEV)
    ops.log_softmax(logits, V, out=ctc.lp)
    st = ops.BeamState(B, beam, 8, DEV)
    st.init()
    ctc.init(in_len)
    out_val = torch.zeros(B, beam, device=DEV)
    out_idx = torch.zeros(B, beam, dtype=torch.int32, device=DEV)
    for step in range(5):
        ids = torch.stack([y[:, step], torch.full((B,), EOS), (y[:, step] - 2 + 1) % (V - 2) + 2, (y[:, step] - 2 + 2) % (V - 2) + 2], 1)
        ctc.cand_id.copy_(ids.int())
        ctc.cand_val.zero_()
        ctc.score(st, in_len, 0.5, out_val, out_idx)
        if step in (0, 3):
            tgt = torch.cat((y[:, :step], torch.full((B, 1), EOS)), 1).to(DEV)
            tl = torch.full((B,), step + 1, dtype=torch.int32, device=DEV)
            _, nll, _ = ops.ctc_loss(logits, B, T, V, in_len, tgt, tl)
            assert bool(((ctc.psi_cand[:, 1] + nll).abs() <= 2e-4 * nll.abs().clamp_min(1.0)).all()), (step, ctc.psi_cand[:, 1], nll)
        st.par_hist[step].copy_(torch.arange(B, dtype=torch.int32))
        st.tok_hist[step].copy_(y[:, step].int())
        st.last_tok.copy_(y[:, step])
        st.ctrl[0] = step + 1
        ctc.advance(st, in_len)


# ------------------------------------------------------------------------------------------------ the search
LOCKSTEP_SEED = 6


@pytest.mark.parametrize('with_lm', [False, True])
def test_joint_search_lockstep_with_the_restatement(with_lm):
    """Eager BeamDecoder with the CTC term against JointSearch fed the GPU's attention (and LM) log-probs and the GPU's CTC
    log-probs, computing its own prefix scores in float64: the same prefixes at every step, scores within 1e-3.  Every
    decision of the committed seed is taken by a margin above 1e-3, so the equality is neither vacuous nor luck."""
    model = _joint_model()
    B, beam, P, max_len, w = 2, 3, 6, 6, 0.3
    lmw = 0.3 if with_lm else 0.0
    lm = None
    if with_lm:
        from opentransformer_b200.lm import TransformerLanguageModel
        torch.manual_seed(77)
        lm = TransformerLanguageModel(dict(vocab_size=4234, num_blocks=2, d_model=256, n_heads=4, d_ff=1024, residual_dropout=0.0,
                                           smoothing=0.1, share_embedding=True)).eval().to(DEV)
    x, mask = _inputs(B, 160, [160, 131], seed=LOCKSTEP_SEED)
    V = model.decoder.vocab_size
    margins = []
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x, mask)
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False, keep_logp=True, ctc=(model.assistor, w, P))
        assert not bd.persistent
        bd.setup(mem, lens)
        bd.lm_weight = lmw
        js = cpr.JointSearch(bd.ctc.lp.view(B, T2, V).cpu(), lens.cpu().tolist(), beam, P, w, lmw)
        for s in range(max_len):
            lm_cpu = None
            if with_lm:
                bd.lm_logp = lm_log_probs(lm, bd.state.reconstruct(s))
                lm_cpu = bd.lm_logp.cpu()
            bd._step_kernels()
            att = bd.logp.cpu().double() - (lmw * lm_cpu.double() if with_lm else 0.0)   # the fused kernel stores att + lmw lm
            margins.append(js.step(att, lm_cpu))
            assert torch.equal(bd.state.reconstruct(s + 1).cpu(), js.preds), f'prefixes differ at step {s}'
            got, want = bd.state.scores.cpu().double(), js.scores.view(-1)
            assert torch.equal(torch.isfinite(got), torch.isfinite(want)), s
            assert float((got - want)[torch.isfinite(want)].abs().max()) < 1e-3, s
    print('lockstep margins', [f'{m:.3e}' for m in margins])
    assert min(margins) > 1e-3, margins


def test_graph_equals_eager_and_early_end():
    model = _joint_model()
    B, beam, max_len = 4, 5, 10
    x, mask = _inputs(B, 240, [240, 200, 111, 239])
    kw = dict(ctc_weight=0.3, beam_width=beam, nbest=2, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    rec_g = SpeechToTextRecognizer(model, **kw)
    rec_e = SpeechToTextRecognizer(model, use_graph=False, **kw)
    p1, s1, n1 = rec_e.recognize_ids(x, mask)
    p2, s2, n2 = rec_g.recognize_ids(x, mask)
    p3, s3, n3 = rec_g.recognize_ids(x, mask)               # the second call replays the captured step
    bd = next(iter(rec_g._decoders.values()))
    assert bd.graph is not None and bd.ctc is not None and not bd.persistent
    assert n1 == n2 == n3 == max_len
    assert torch.equal(p1, p2) and torch.equal(p2, p3) and torch.equal(s1, s2) and torch.equal(s2, s3)
    assert bool(torch.isfinite(s1).all())
    # the CTC term is in the scores: an attention-only recognizer of the same model scores differently
    _, s0, _ = SpeechToTextRecognizer(model, **dict(kw, ctc_weight=0.0)).recognize_ids(x, mask)
    assert not torch.equal(s0, s1)
    # a decoder eager to end: both paths stop at the same step, before max_len
    model2 = _joint_model(eos_bias=1e4)
    kw['max_len'] = 24
    q1, t1, m1 = SpeechToTextRecognizer(model2, use_graph=False, **kw).recognize_ids(x, mask)
    q2, t2, m2 = SpeechToTextRecognizer(model2, **kw).recognize_ids(x, mask)
    assert m1 == m2 < 24, (m1, m2)
    assert torch.equal(q1, q2) and torch.equal(t1, t2)


def test_the_ctc_term_recovers_what_the_decoder_ranks_second():
    """A decoder whose output layer is its bias alone: a decoy token first, the tokens of y and <S/E> next, the rest far
    behind; CTC log-probs peaked on an alignment of y <S/E>.  Attention-only decoding never starts with y (without a length
    penalty its 1-best is the bare <S/E>); at ctc_weight 0.9 the 1-best is y <S/E>."""
    model = _joint_model(n_dec=1)
    y, decoy = [50, 50, 70, 30], 99
    with torch.no_grad():
        model.decoder.output_layer.weight.zero_()           # tied to the embedding: the decoder sees positions only
        model.decoder.output_layer.bias.zero_()
        model.decoder.output_layer.bias[decoy] = 3.0
        for v in set(y) | {EOS}:
            model.decoder.output_layer.bias[v] = 2.0
    B, beam, P, max_len, V = 1, 3, 6, 8, model.decoder.vocab_size
    x, mask = _inputs(B, 160, [160])
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x, mask)
        frames = [50, 0, 50, 0, 70, 0, 30, 0, EOS]
        lp = torch.full((T2, V), -30.0)
        for t in range(T2):
            lp[t, frames[t] if t < len(frames) else 0] = 0.0
        lp = torch.log_softmax(lp, dim=-1)
        best = {}
        for w in (0.0, 0.9):
            bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False,
                             ctc=(model.assistor, w, P) if w else None)
            bd.setup(mem, lens)
            if w:
                bd.ctc.lp.copy_(lp)                          # in place of the head's output
                bd.ctc.init(bd.mem_len)
            steps = bd.run(max_len)
            preds, _ = bd.state.finalize(0.0, 5, 1)
            best[w] = preds[0, 0, :steps].tolist()
    assert best[0.0][:len(y) + 1] != y + [EOS] and best[0.0][0] != y[0]
    assert best[0.9][:len(y) + 1] == y + [EOS], best


def test_weight_zero_is_todays_path():
    """On the benchmark geometry: no CTC buffer, the persistent decode kernel still chosen, ids and scores those of a
    recognizer built without the argument."""
    model = _joint_model(n_enc=1, n_dec=1)
    B, T = 32, 1000
    x, mask = _inputs(B, T, [T - 7 * b for b in range(B)])
    kw = dict(beam_width=10, nbest=1, max_len=60, penalty=0.6, lamda=5, ngpu=1)
    rec0 = SpeechToTextRecognizer(model, ctc_weight=0.0, **kw)
    rec = SpeechToTextRecognizer(model, **kw)
    p0, s0, n0 = rec0.recognize_ids(x, mask)
    p, s, n = rec.recognize_ids(x, mask)
    bd = next(iter(rec0._decoders.values()))
    assert bd.ctc is None and bd.persistent
    assert n0 == n and torch.equal(p0, p) and torch.equal(s0, s)


@pytest.mark.parametrize('w', [0.0, 0.3])
def test_recognize_spans(w):
    """The ids, scores and steps of recognize_ids, and ops.ctc_align called by hand on the 1-best plus its closing <S/E>;
    spans lie inside the utterance and follow one another."""
    model = _joint_model()
    B, max_len = 3, 6
    x, mask = _inputs(B, 240, [240, 170, 131])
    rec = SpeechToTextRecognizer(model, ctc_weight=w, beam_width=4, nbest=2, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    ids, sc, n = rec.recognize_ids(x, mask)
    ids2, sc2, n2, spans = rec.recognize_spans(x, mask)
    assert n == n2 and torch.equal(ids, ids2) and torch.equal(sc, sc2)
    assert spans.shape == (B, n + 1, 2) and spans.dtype == torch.int32
    V = model.decoder.vocab_size
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x, mask)
        lp = ops.log_softmax(model.assistor.logits_bf16(mem), V).view(B, T2, V)
    tgt = torch.cat((ids[:, 0], torch.full((B, 1), EOS, dtype=torch.int64, device=DEV)), 1)
    n_tok = [row.index(EOS) + 1 for row in tgt.cpu().tolist()]
    _, _, want, path = ops.ctc_align(lp, lens, tgt, torch.tensor(n_tok, dtype=torch.int32, device=DEV))
    assert torch.equal(spans, want) and bool(torch.isfinite(path).all())
    sp, lens = spans.cpu(), lens.cpu()
    for b in range(B):
        k = n_tok[b]
        assert bool((sp[b, k:] == -1).all())
        assert bool((sp[b, :k, 0] >= 0).all()) and bool((sp[b, :k, 1] <= int(lens[b])).all())
        assert bool((sp[b, :k, 0] < sp[b, :k, 1]).all()) and bool((sp[b, 1:k, 0] >= sp[b, :k - 1, 1]).all())
