"""GPU checks of ancestral sampling and sampling-based MWER training (DESIGN.md 4.11) against the float64 restatement
(tests/mwer_sample_ref.py): otb_sample_step row by row (tokens, score increments, ended rows, the search state's
conventions, ties across warps, canaries past V), the distribution of its draws, seeds and graph replay of the sampling
decoder, sample_ids against a float64 decoder fed the same uniforms, otb_mwer_sample_coeff, the sampled MWER pass against
the fp32 oracle, and FusedTrainer(mwer_samples=4).  Each case prints its errors."""
import ctypes

import numpy as np
import pytest
import torch

from tests import mwer_ref as mr
from tests import mwer_sample_ref as sr

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import _lib, ops, train
    from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer, second_pass_rows
    DEV = torch.device('cuda:0')

from oracle import speech_model as om

EOS = 1
TIE = 2.0 ** 30       # x + g rounds to exactly 2^30 in fp32 for every Gumbel value (|g| < 17 < half an ulp of 2^30)


def _gumbel_bound(x, g):
    """What the fp32 perturbed value x + g can differ from float64 by: two accurate logf (1 ulp each, the inner one's
    relative error carried through the outer log) and the rounding of the sum."""
    return 4e-7 + 2.4e-7 * (np.abs(x) + 2.0 * np.abs(g))


def _state(B, K, Lmax):
    st = ops.BeamState(B, K, Lmax, DEV)
    st.init()
    return st


def _tie_rows(V):
    """(row, lower id, higher id) of the rows whose two largest logits tie exactly after perturbation: the pair in
    different threads of one warp, in different warps with the lower id in the later warp, and in the same thread."""
    rows = []
    if V >= 3:
        rows.append((5, V // 3, V - 1))
    if V >= 512:
        rows += [(6, 100, 300), (7, 65, 321)]      # warp 3 vs warp 1; thread 65 twice
    return rows


@pytest.mark.parametrize('V', [1, 2, 5, 31, 257, 4234, 49152])
def test_sample_step_matches_the_restatement(V):
    B, K, Lmax, step = 3, 4, 6, 2
    N = B * K
    g = torch.Generator().manual_seed(V)
    ld = (V + 3) // 4 * 4 + 4
    x = torch.randn(N, V, generator=g) * 3.0
    x[1, ::3] = float('-inf')                       # -inf entries (token 0 among them)
    if V > 1:
        x[1, V - 1] = 0.5                          # a finite entry even at V = 2
    x[2, V // 2] += 25.0                            # a peaked row
    if V > EOS:
        x[8, EOS] = 60.0                            # a row that draws <S/E> and ends
    ties = _tie_rows(V)
    for r, a, b in ties:
        x[r, a] = x[r, b] = TIE
    logits = torch.full((N, ld), float('nan'))
    logits[:, :V] = x
    logits = logits.to(DEV)
    before = logits.clone()
    st = _state(B, K, Lmax)
    flag = torch.zeros(N, dtype=torch.bool)
    flag[[3, 4]] = True                              # ended rows
    scores0 = torch.randn(N, generator=g)
    anc_cur = torch.randint(0, N, (N, Lmax), generator=g, dtype=torch.int32)
    st.flag.copy_(flag.to(torch.uint8))
    st.scores.copy_(scores0)
    st.ctrl[0] = step
    st.anc[step & 1].copy_(anc_cur)
    seed_val = -123456 + V
    ops.sample_step(logits, V, st, torch.tensor([seed_val], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    assert torch.equal(torch.isnan(logits), torch.isnan(before)) and torch.equal(logits[:, :V], before[:, :V])
    tok = st.tok_hist[step].cpu()
    sc = st.scores.cpu()
    x64 = x.double().numpy()
    checked = ambiguous = 0
    worst_inc = 0.0
    for n in range(N):
        if flag[n]:
            assert int(tok[n]) == EOS and float(sc[n]) == float(scores0[n]), f'ended row {n}'
            continue
        if not np.isfinite(x64[n]).any():           # nothing to draw: token 0 and score -inf
            assert int(tok[n]) == 0 and float(sc[n]) == float('-inf'), f'row {n} without a finite logit'
            continue
        t64, _, z = sr.draw(x64[n], seed_val, step, n)
        fin = np.isfinite(z)
        gum = np.where(fin, z - np.where(fin, x64[n], 0.0), 0.0)
        order = np.argsort(-z[fin], kind='stable')
        if fin.sum() >= 2:
            gap = z[fin][order[0]] - z[fin][order[1]]
            bound = 2.0 * float(_gumbel_bound(x64[n][fin], gum[fin]).max())
        else:
            gap, bound = np.inf, 0.0
        if any(r == n for r, _, _ in ties):
            lo = next(a for r, a, _ in ties if r == n)
            assert int(tok[n]) == lo, f'row {n}: an exact tie must go to the lower id {lo}, got {int(tok[n])}'
        elif gap > bound:
            assert int(tok[n]) == t64, f'row {n}: token {int(tok[n])} vs float64 {t64} (gap {gap:.3e} > bound {bound:.3e})'
            checked += 1
        else:
            ambiguous += 1
        # the increment of the device's own token, against float64
        t = int(tok[n])
        xf = x64[n][np.isfinite(x64[n])]
        lse = xf.max() + np.log(np.exp(xf - xf.max()).sum())
        inc64 = x64[n][t] - lse
        err = abs(float(sc[n]) - (float(scores0[n]) + inc64))
        lim = 2e-6 * (abs(x64[n][t]) + abs(lse)) + 2e-5 + 1e-6 * abs(float(scores0[n]))
        assert err <= lim, f'row {n}: score increment off by {err:.3e} (bound {lim:.3e})'
        worst_inc = max(worst_inc, err / lim)
    ended = (tok == EOS) | flag
    assert torch.equal(st.flag.cpu().bool(), ended)
    assert torch.equal(st.last_tok.cpu(), tok.long())
    assert torch.equal(st.par_hist[step].cpu(), torch.arange(N, dtype=torch.int32))
    nxt = st.anc[(step & 1) ^ 1].cpu()
    assert torch.equal(nxt[:, :step], anc_cur[:, :step]) and torch.equal(nxt[:, step], torch.arange(N, dtype=torch.int32))
    assert st.ctrl.cpu().tolist() == [step + 1, int(bool(ended.all())), 0, 0]
    if V > EOS:
        assert int(tok[8]) == EOS
    print(f'sample_step V={V}: {checked} tokens equal float64 past the margin, {ambiguous} within it, ties {len(ties)}; '
          f'worst score increment {worst_inc:.2f} of its bound')


def test_sample_step_ends_the_search_and_then_freezes():
    V, B, K, Lmax = 5, 2, 3, 4
    x = torch.randn(B * K, V) * 3.0
    x[:, EOS] = 60.0
    logits = x.to(DEV)
    st = _state(B, K, Lmax)
    seed = torch.tensor([7], dtype=torch.int32, device=DEV)
    ops.sample_step(logits, V, st, seed)
    assert st.ctrl.cpu().tolist() == [1, 1, 0, 0] and bool((st.tok_hist[0] == EOS).all())
    snap = [t.clone() for t in (st.tok_hist, st.par_hist, st.scores, st.flag, st.anc, st.ctrl)]
    ops.sample_step(logits, V, st, seed)
    for a, b in zip(snap, (st.tok_hist, st.par_hist, st.scores, st.flag, st.anc, st.ctrl)):
        assert torch.equal(a, b), 'a step after the end must leave the state as it was'


def test_sample_step_refusals():
    st = _state(1, 2, 4)
    seed = torch.zeros(1, dtype=torch.int32, device=DEV)
    big = torch.zeros(2, 49156, device=DEV)
    with pytest.raises(ValueError, match='sample_step'):
        ops.sample_step(big, 49153, st, seed)
    lib = _lib.lib()
    for V, state in ((49153, st), (0, st), (4, _lib.BeamStateC(*([None] * 7), 0, 1, 4))):
        c = state.c if hasattr(state, 'c') else state
        assert lib.otb_sample_step(big.data_ptr(), 49156, V, ctypes.byref(c), seed.data_ptr(), None) != 0
        assert lib.otb_last_error().decode().startswith('otb_sample_step')


def _chi_square(counts, p, min_expected=5.0):
    """Pearson's statistic over the bins with at least min_expected expected draws, the rest pooled into one bin."""
    from scipy.stats import chi2
    n = counts.sum()
    e = p * n
    big = e >= min_expected
    obs = np.append(counts[big], counts[~big].sum())
    exp = np.append(e[big], e[~big].sum())
    keep = exp > 0
    stat = float(((obs[keep] - exp[keep]) ** 2 / exp[keep]).sum())
    dof = int(keep.sum()) - 1
    return stat, dof, float(chi2.ppf(0.999, dof))


@pytest.mark.parametrize('kind', ['peaked', 'flat'])
def test_sample_step_distribution(kind):
    """10^5 draws at a fixed seed (1000 rows x 100 steps, every row reset to live before each step) against softmax(x):
    Pearson's chi-square under its 0.999 quantile.  The seed is fixed, so the test is deterministic."""
    g = torch.Generator().manual_seed(5)
    if kind == 'peaked':
        V = 4234
        x = torch.randn(V, generator=g) * 2.0
        x[17] += 9.0
    else:
        V = 5
        x = torch.randn(V, generator=g) * 0.1
    rows, steps = 1000, 100
    st = _state(rows, 1, steps)
    st.scores.zero_()
    logits = x.view(1, V).expand(rows, V).contiguous().to(DEV)
    seed = torch.tensor([99], dtype=torch.int32, device=DEV)
    for _ in range(steps):
        st.flag.zero_()
        st.ctrl[1] = 0
        ops.sample_step(logits, V, st, seed)
    counts = torch.bincount(st.tok_hist.cpu().view(-1).long(), minlength=V).double().numpy()
    p = torch.softmax(x.double(), 0).numpy()
    stat, dof, lim = _chi_square(counts, p)
    top = int(np.argmax(p))
    print(f'{kind} row V={V}: chi-square {stat:.1f} on {dof} dof (0.999 quantile {lim:.1f}); token {top}: '
          f'{int(counts[top])} draws, expected {p[top] * counts.sum():.0f}')
    assert counts.sum() == rows * steps and stat < lim


# ------------------------------------------------------------------------------------------------ the sampling decoder
def _model(seed=1234):
    from tests.test_gpu_train import _build, _params
    params = _params(n_enc=1, n_dec=2, tied=False)
    model, sd = _build(params, seed)
    return model.eval(), params


def _inputs(B=3):
    from tests.test_gpu_train import _batch
    x, mask, _ = _batch(B=B, lens=(200, 160, 181)[:B])
    return x.to(DEV), mask.to(DEV)


def _decode(bd, mem, mem_len, seed, steps, use_logits=False):
    bd.setup(mem, mem_len)
    bd.seed.fill_(seed)
    trace = []
    for s in range(steps):
        bd.step()
        trace.append((bd.state.tok_hist[:s + 1].clone(), bd.state.scores.clone(), bd.logits[:, :bd.dec.vocab_size].clone()
                      if use_logits else None))
    return trace


def test_sampling_decoder_seeds_and_graph_replay():
    """Same seed, same ids; a new seed, new ids; the captured step replayed equals the eager step, step by step."""
    model, _ = _model()
    rec = SpeechToTextRecognizer(model, max_len=12)
    x, mask = _inputs()
    with torch.no_grad():
        mem, mem_len, B, T2 = rec._encode_bf16(x, mask)
        K, L = 4, 12
        eager = _decode(BeamDecoder(model.decoder, B, K, T2, L, DEV, use_graph=False, sample=True), mem, mem_len, 31, L)
        bd_g = BeamDecoder(model.decoder, B, K, T2, L, DEV, use_graph=True, sample=True)
        graph = _decode(bd_g, mem, mem_len, 31, L)
        assert bd_g.graph is not None and not bd_g.persistent
        for s, ((te, se, _), (tg, sg, _)) in enumerate(zip(eager, graph)):
            assert torch.equal(te, tg) and torch.equal(se, sg), f'graph replay differs from eager at step {s}'
        again = _decode(bd_g, mem, mem_len, 31, L)
        assert all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) for a, b in zip(graph, again))
        other = _decode(bd_g, mem, mem_len, 32, L)
        differ = int((other[-1][0] != graph[-1][0]).sum())
        print(f'sampling decoder: graph == eager over {L} steps; seed 32 vs 31: {differ} of {graph[-1][0].numel()} tokens differ')
        assert differ > 0
        ids1, _, _ = rec.sample_ids(x, mask, K, 31)
        ids2, _, _ = rec.sample_ids(x, mask, K, torch.tensor([31], dtype=torch.int32, device=DEV))
        assert torch.equal(ids1, ids2)
        assert torch.equal(ids1[:, :, :1], graph[0][0][0].view(B, K, 1).long())


def test_sample_ids_against_a_float64_decoder():
    """sample_ids, then the same samples drawn step by step by the eager sampling decoder (bit-identical), with the
    float64 oracle decoder teacher-forced on each sample's prefix and fed the same uniforms.  Where the float64 perturbed
    top-two gap exceeds twice the row's largest |log-prob error| of the bf16 decoder (plus the fp32 bound of g), the token
    must equal the float64 draw; the rest are reported.  Each sample's log-prob is within the sum of its rows' errors of
    the float64 sum."""
    from opentransformer_b200 import modules
    model, params = _model()
    with torch.no_grad():
        model.decoder.output_layer.bias[EOS] += 6.0       # <S/E> likely enough that samples end inside max_len
    modules.bump_param_generation()
    K, L, seed = 4, 10, 2024
    rec = SpeechToTextRecognizer(model, max_len=L)
    x, mask = _inputs()
    V = model.decoder.vocab_size
    with torch.no_grad():
        ids, lens, lp = rec.sample_ids(x, mask, K, seed)
        mem, mem_len, B, T2 = rec._encode_bf16(x, mask)
        steps = ids.shape[2]
        assert ids.shape == (B, K, steps) and lens.shape == (B, K) and lp.shape == (B, K)
        assert torch.equal(lens, (ids != EOS).sum(dim=2, dtype=torch.int32))
        trace = _decode(BeamDecoder(model.decoder, B, K, T2, L, DEV, use_graph=False, sample=True), mem, mem_len, seed, steps,
                        use_logits=True)
        assert torch.equal(trace[-1][0][:steps].t().reshape(B, K, steps).long(), ids), 'eager and sample_ids differ'
        assert torch.equal(trace[-1][1].view(B, K), lp)
        sd64 = {f'decoder.{k}': v.detach().double() for k, v in model.decoder.state_dict().items()}
        kw = om.decoder_kwargs(params)
        mem64 = mem.double().view(B, T2, -1)
        mmask = torch.arange(T2, device=DEV)[None] < mem_len[:, None]
        N = B * K
        flat = ids.view(N, steps).cpu()
        preds = torch.cat((torch.full((N, 1), EOS, dtype=torch.long), flat), dim=1)
        lp64 = torch.zeros(N, dtype=torch.float64)
        err_sum = torch.zeros(N, dtype=torch.float64)
        checked = ambiguous = 0
        worst = 0.0
        for s in range(steps):
            live = (flat[:, :s] != EOS).all(dim=1) if s else torch.ones(N, dtype=torch.bool)
            rows = live.nonzero().view(-1)
            if rows.numel() == 0:
                break
            with torch.device(DEV):
                ref = om.decoder_inference(preds[rows, :s + 1].to(DEV), mem64[rows.to(DEV) // K], mmask[rows.to(DEV) // K],
                                           sd64, 'decoder.', **kw).cpu()
            got = torch.log_softmax(trace[s][2][rows].double(), dim=-1).cpu()
            delta = (got - ref).abs().max(dim=1).values
            worst = max(worst, float(delta.max()))
            for i, n in enumerate(rows.tolist()):
                r = ref[i].numpy()
                z = r + sr.gumbel(sr.uniforms(seed, s, n, V))
                top2 = np.partition(z, -2)[-2:]
                gap = top2[1] - top2[0]
                bound = 2 * float(delta[i]) + 2 * float(_gumbel_bound(np.abs(r).max(), 17.0))
                tok = int(flat[n, s])
                if gap > bound:
                    assert tok == int(np.argmax(z)), f'sample {n} step {s}: token {tok} vs float64 {int(np.argmax(z))}'
                    checked += 1
                else:
                    ambiguous += 1
                lp64[n] += float(r[tok])
                err_sum[n] += float(delta[i])
        diff = (lp.view(-1).cpu().double() - lp64).abs()
        print(f'sample_ids (B={B}, K={K}, {steps} steps, lengths {lens.tolist()}): {checked} tokens equal the float64 draw, '
              f'{ambiguous} inside the margin; |log-prob error| of a row <= {worst:.3e}; sample log-prob vs float64 '
              f'{float(diff.max()):.3e} (bound {float(err_sum.max()):.3e})')
        assert checked > 0 and bool((diff <= err_sum + 1e-4).all())


# ------------------------------------------------------------------------------------------------ the sampled estimator
@pytest.mark.parametrize('scale_on_device', [False, True])
def test_mwer_sample_coeff_matches_float64(scale_on_device):
    g = torch.Generator().manual_seed(3)
    B, K = 5, 7
    err = torch.randint(0, 30, (B, K), generator=g, dtype=torch.int32)
    err[2] = 11                                               # all W equal: exactly zero
    scale = 0.25 / B
    if scale_on_device:
        loss, coeff = ops.mwer_sample_coeff(err.to(DEV), 0.5 / B, torch.tensor(0.5, device=DEV))
    else:
        loss, coeff = ops.mwer_sample_coeff(err.to(DEV), scale)
    mean, c = sr.sample_coefficients(err.double(), B, grad_scale=0.25)
    print(f'mwer_sample_coeff: loss max err {float((loss.cpu().double() - mean).abs().max()):.2e}, coeff max err '
          f'{float((coeff.cpu().double() - c).abs().max()):.2e}')
    torch.testing.assert_close(loss.cpu().double(), mean, rtol=1e-6, atol=0)
    torch.testing.assert_close(coeff.cpu().double(), c, rtol=1e-5, atol=1e-9)
    assert bool((coeff[2] == 0).all())


def _fixed_samples(tgt, K, seed):
    """Rows [B, K, 6] as sample_ids returns them: utterance 0 holds a repeated sample (kept: samples are drawn with
    replacement), one row reaches the width without <S/E>, and utterance 2's samples are all the same sequence, so its W
    are equal and its MWER gradient is exactly zero."""
    from tests.test_gpu_mwer import _fixed_nbest
    ids = _fixed_nbest(tgt, K, seed)
    ids[2] = ids[2, 1]
    return ids


def test_sampled_mwer_pass_matches_oracle():
    """forward_backward(mwer_estimator='sample') on fixed rows: the loss is mean_b W^_b + lambda L_CE, and every gradient
    against the fp32 oracle with the sampled coefficients c_k = (W_k - W^_b) / (K B) held fixed, within the bounds of the
    n-best pass (tests/test_gpu_mwer.py).  An utterance whose W are equal gets exactly zero coefficients and rows of
    dlogits."""
    from tests.test_gpu_mwer import REL_L2_MWER, REL_L2_MWER_ALL, REL_L2_MWER_LAST_NORM_BIAS, _oracle_mwer, _rel
    from tests.test_gpu_train import _batch, _build, _params
    params = _params(n_enc=2, n_dec=2)
    model, sd = _build(params)
    x, mask, tgt = _batch()
    tlen = (tgt[:, 1:] != 0).sum(1).to(torch.int32)
    B, K, lam = x.shape[0], 4, 0.3
    ids = _fixed_samples(tgt, K, seed=3)
    hyp_in, hyp_tgt, n, Lp = second_pass_rows(ids.to(DEV))
    hyps = [[mr.cut(ids[b, k]) for k in range(K)] for b in range(B)]
    refs = [mr.reference(tgt[b], tlen[b]) for b in range(B)]
    W = torch.tensor([[mr.edit_distance(y, refs[b]) for y in hyps[b]] for b in range(B)], dtype=torch.float64)
    assert len(set(W[2].tolist())) == 1 and len(set(W[0].tolist())) > 1
    mean, coeff = sr.sample_coefficients(W, B)
    seed = torch.tensor([777], dtype=torch.int32, device=DEV)
    _, g_ref = _oracle_mwer(x, mask, tgt, tlen, sd, params, hyp_in.cpu(), hyps, K, lam, False, coeff=coeff)
    with torch.no_grad():
        loss, g = train.forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV),
                                         drop_seed=seed, nbest=(hyp_in, hyp_tgt.view(B * K, Lp), K), mwer_ce_weight=lam,
                                         mwer_estimator='sample')
        ce, _ = train.forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV),
                                       want_grads=False, drop_seed=seed)
        # the product's own coefficients and gradient rows for the equal-W utterance
        err = ops.edit_distance(hyp_tgt.view(B * K, Lp), n.view(-1), tgt[:, 1:].to(torch.int32).to(DEV),
                                (tlen - 1).to(DEV), K)
        _, c_dev = ops.mwer_sample_coeff(err.view(B, K), 1.0 / B)
    want = float(mean.mean()) + lam * float(ce)
    print(f'sampled MWER pass: loss gpu {float(loss):.6f}, mean W^ + lambda CE {want:.6f}; coefficients {c_dev.tolist()}')
    assert abs(float(loss) - want) <= 1e-5 * abs(want)
    assert bool((c_dev[2] == 0).all()) and float(c_dev.abs().max()) > 1e-2
    names = [n for n in g_ref if g_ref[n] is not None]
    last_bias = f'decoder.blocks.{params["decoder"]["n_blocks"] - 1}.norm3.bias'

    def scaled(n):
        return _rel(g[n], g_ref[n]) * (REL_L2_MWER / REL_L2_MWER_LAST_NORM_BIAS if n == last_bias else 1.0)
    worst = sorted(((scaled(n), n) for n in names), reverse=True)
    r_all = _rel(torch.cat([g[n].reshape(-1).cpu() for n in names]), torch.cat([g_ref[n].reshape(-1) for n in names]))
    print(f'  gradients vs oracle: all rel_l2 {r_all:.3e}; worst ' + ', '.join(f'{n} {r:.2e}' for r, n in worst[:3]))
    assert r_all < REL_L2_MWER_ALL and worst[0][0] < REL_L2_MWER, worst[:3]
    # the MWER gradient rows of the equal-W utterance are exactly zero
    with torch.no_grad():
        logits = torch.randn(B * K * Lp, model.decoder.ld_logits, device=DEV)
        flat = hyp_tgt.reshape(-1).to(torch.int32).contiguous()
        tok = ops.token_logprob(logits, model.decoder.vocab_size, flat)
        d = ops.mwer_grad(logits, model.decoder.vocab_size, flat, tok, c_dev)
    assert float(d[2 * K * Lp:3 * K * Lp].float().abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ FusedTrainer
def _trainer(use_graph, seed=1234, accum_steps=1):
    """FusedTrainer(mwer_samples=4) on an untied model whose samples carry a gradient.  With the tied embedding <S/E> is the
    near-certain first draw, so every sample is the bare <S/E>; untied, <S/E> is a 2e-4 draw, so every sample runs to
    max_len with random tokens and its edit distance is the same for all K.  Either way every coefficient is 0.  The
    <S/E> logit raised by 6 ends samples at varied lengths around the references' 5 to 10 tokens, so W varies."""
    from opentransformer_b200 import modules
    from tests.test_gpu_train import _build, _params
    model, _ = _build(_params(n_enc=1, n_dec=1, tied=False), seed)
    with torch.no_grad():
        model.decoder.output_layer.bias[EOS] += 6.0
    modules.bump_param_generation()
    tr = train.FusedTrainer(model.train(), clip_grad=0.05, use_graph=use_graph, mwer_samples=4, mwer_max_len=12,
                            accum_steps=accum_steps)
    tr.graph_after = 1
    rows = []
    decode = tr._with_nbest

    def recording(batch):                   # the sampled rows (targets i32 [B*K, Lp]) each micro-step hands to the pass
        out = decode(batch)
        rows.append(out[-1].clone())
        return out
    tr._with_nbest = recording
    return model, tr, rows


def _cross_entropy(model, x, mask, tgt):
    """L_CE of the training pass without MWER on the model's current weights (every dropout rate is 0)."""
    with torch.no_grad():
        return float(train.forward_backward(model.train(), x, mask, tgt, want_grads=False)[0])


def _expected_loss(ce, rows, tgt, K, lam):
    """mean_b mean_k W_k + lambda * L_CE of the sampled rows (targets [B*K, Lp], -1 after y <S/E>), the references cut at
    the transcript's first <S/E> as the trainer cuts them without truth_length -> (loss, W float64 [B, K])."""
    B = tgt.shape[0]
    r, t = rows.cpu(), tgt.cpu()
    hyps = [r[i, :int((r[i] >= 0).sum()) - 1].tolist() for i in range(B * K)]
    refs = [t[b, 1:][:int((t[b, 1:] == EOS).int().argmax())].tolist() for b in range(B)]
    W = torch.tensor([[mr.edit_distance(hyps[b * K + k], refs[b]) for k in range(K)] for b in range(B)], dtype=torch.float64)
    return float(W.mean(dim=1).mean()) + lam * ce, W


def test_fused_trainer_sampled_mwer():
    """On samples that are not trivial (Lp > 1, an utterance with unequal W, so some coefficient is not 0): each step's loss
    is mean_b W^_b + lambda L_CE of the rows it sampled; consecutive micro-steps draw new rows; graph and eager draw the same
    rows and give the same losses; the MWER term changes the gradient (against lambda times the cross-entropy gradient alone);
    a state_dict round trip resumes with the same seed, so the resumed step draws the same rows and gives the same loss.
    Without mwer_samples the saved keys are as before."""
    from opentransformer_b200 import modules
    from tests.test_gpu_train import _batch
    x, mask, tgt = (t.to(DEV) for t in _batch())
    K, lam = 4, 0.01
    runs = []
    for use_graph in (False, True):
        model, tr, rows = _trainer(use_graph)
        p0 = tr.flat_p.clone()
        losses = []
        for _ in range(2):
            ce = _cross_entropy(model, x, mask, tgt)
            losses.append(float(tr.step(x, mask, tgt)))
            want, W = _expected_loss(ce, rows[-1], tgt, K, lam)
            print(f'  graph={use_graph}: Lp {rows[-1].shape[1]}, W {W.tolist()}, loss {losses[-1]:.6f}, '
                  f'mean W^ + lambda CE {want:.6f}')
            assert rows[-1].shape[1] > 1 and any(len(set(w)) > 1 for w in W.tolist()), 'the samples must carry a gradient'
            assert abs(losses[-1] - want) <= 1e-5 * abs(want)
        assert rows[0].shape != rows[1].shape or not torch.equal(rows[0], rows[1]), 'the seed must advance'
        assert model.training and bool(torch.isfinite(tr.flat_p).all())
        runs.append((losses, tr.flat_p.clone(), len(tr._graphs), float((tr.flat_p - p0).abs().max()), rows))
    print('sampled MWER FusedTrainer losses: eager', runs[0][0], 'graph', runs[1][0], '; largest weight change', runs[0][3])
    assert runs[1][2] >= 1 and runs[0][0] == runs[1][0] and runs[0][3] > 0.0
    assert all(torch.equal(a, b) for a, b in zip(runs[0][4], runs[1][4])), 'graph and eager sampled different rows'
    # the order of the fp32 atomics that add the embedding gradient may differ: far less than one Adam step (lr(3) = 1.4e-7)
    assert float((runs[0][1] - runs[1][1]).abs().max()) < 1.4e-7
    # the gradient of one micro-step (accumulation 2 keeps it in flat_g) against lambda times the cross-entropy gradient
    model, tr, rows = _trainer(False, accum_steps=2)
    with torch.no_grad():
        _, g_ce = train.forward_backward(model.train(), x, mask, tgt)
    tr.step(x, mask, tgt)
    g = tr.flat_g * 2.0
    ce_part = torch.zeros_like(g)
    for n, (o, k) in tr.offsets.items():
        if g_ce.get(n) is not None:
            ce_part[o:o + k] = lam * g_ce[n].reshape(-1)
    share = float((g - ce_part).norm() / g.norm())
    print(f'micro-step gradient: |g - lambda g_CE| / |g| = {share:.3f}')
    assert share > 0.1, 'the MWER term must change the gradient'
    # resume
    model, tr, rows = _trainer(False)
    tr.step(x, mask, tgt)
    sd, weights = tr.state_dict(), tr.flat_p.clone()
    assert 'sample_seed' in sd['fused_trainer']
    want = float(tr.step(x, mask, tgt))
    model2, tr2, rows2 = _trainer(False, seed=99)
    tr2.flat_p.copy_(weights)
    modules.bump_param_generation()
    tr2.load_state_dict(sd)
    assert int(tr2.sample_seed) == sd['fused_trainer']['sample_seed']
    got = float(tr2.step(x, mask, tgt))
    print(f'resumed step: loss {got} vs {want}')
    assert torch.equal(rows2[0], rows[1]) and got == want
    from tests.test_gpu_train import _build, _params
    plain = train.FusedTrainer(_build(_params(n_enc=1, n_dec=1))[0].train(), mwer_nbest=2, use_graph=False)
    assert 'sample_seed' not in plain.state_dict()['fused_trainer']
