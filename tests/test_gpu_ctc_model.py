"""GPU checks of the CTC-only model: the three decoding kernels against the CPU restatement (tests/ctc_ref.py), training
against the fp32 restatement for a Transformer and a Conformer encoder (with replayed dropout masks), FusedTrainer, the
autograd seam, the recogniser end to end, and the SpeechToText micro-step's launch count."""

import pytest
import torch

from tests import ctc_ref

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.model import CTCModel
    from opentransformer_b200.recognize import CTCRecognizer
    DEV = torch.device('cuda:0')

from oracle import train_step as ot

REL_L2_GRAD = 4e-2


def _rel(a, b):
    return float((a.float().cpu() - b.float().cpu()).norm() / (b.float().cpu().norm() + 1e-20))


def _logits(rows, V, seed, scale=3.0):
    """Tie-free fp32 logits [rows, ld] (ld = V padded to 8, junk in the pad columns)."""
    g = torch.Generator().manual_seed(seed)
    ld = (V + 7) // 8 * 8
    x = torch.randn(rows, ld, generator=g) * scale
    x[:, V:] = 1e4                         # must be ignored
    return x.to(DEV)


def _lengths(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.randint(1, T + 1, (B,), generator=g)
    n[0] = T
    return n.to(torch.int32).to(DEV)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize('V', [40, 4234])
@pytest.mark.parametrize('K', [1, 40])
def test_frame_topk_matches_log_softmax_topk(V, K):
    B, T = 4, 37
    x = _logits(B * T, V, seed=V + K)
    n = _lengths(B, T, seed=3)
    lp, ids = ops.ctc_frame_topk(x, B, T, V, n, K)
    ref = torch.log_softmax(x[:, :V].double(), dim=-1)
    rv, ri = ref.topk(K, dim=-1)
    valid = (torch.arange(T, device=DEV)[None] < n[:, None].long()).reshape(-1)
    assert torch.equal(ids[valid].long(), ri[valid])
    torch.testing.assert_close(lp[valid].double(), rv[valid], rtol=0, atol=1e-5)
    assert bool((ids[~valid] == -1).all()) and bool(torch.isinf(lp[~valid]).all())


def test_frame_topk_rows_with_fewer_numbers_than_k():
    """A row with only 3 non-NaN logits (a diverged model) fills ranks 3.. with -1 / -inf, and the decoders never emit -1."""
    V, T, K = 40, 4, 10
    x = _logits(T, V, seed=11)
    x[1, :] = float('nan')
    x[1, [3, 7, 9]] = torch.tensor([1.0, 3.0, 2.0], device=DEV)
    n = torch.tensor([T], dtype=torch.int32, device=DEV)
    lp, ids = ops.ctc_frame_topk(x, 1, T, V, n, K)
    assert ids[1, :3].tolist() == [7, 9, 3] and bool((ids[1, 3:] == -1).all())
    assert bool(torch.isinf(lp[1, 3:]).all()) and bool((lp[1, 3:] < 0).all())
    assert bool((ids[[0, 2, 3]] >= 0).all())
    lp1, ids1 = ops.ctc_frame_topk(torch.full_like(x, float('nan')), 1, T, V, n, 1)
    assert bool((ids1 == -1).all())
    out, nout, _ = ops.ctc_greedy(lp1, ids1, 1, T, n)
    assert int(nout[0]) == 0 and bool((out == 0).all())
    bids, bn, _ = ops.ctc_prefix_beam(lp, ids, 1, T, n, 4)         # the NaN row's log-probs are NaN: nothing survives it
    assert bool((bids >= 0).all()) and bool((bn >= 0).all())


def _greedy_logits(B, T, V, seed):
    """Logits whose best tokens come in runs from a few ids and blanks: repeats, repeats split by blank, blank runs."""
    g = torch.Generator().manual_seed(seed)
    best = torch.randint(0, 4, (B, T), generator=g)
    run = torch.rand(B, T, generator=g) < 0.5
    for t in range(1, T):
        best[:, t] = torch.where(run[:, t], best[:, t - 1], best[:, t])
    x = torch.randn(B * T, (V + 7) // 8 * 8, generator=g)
    x.view(B, T, -1).scatter_(2, best.unsqueeze(2), 6.0)
    return x.to(DEV)


@pytest.mark.parametrize('B', [1, 32])
@pytest.mark.parametrize('T', [1, 7, 249])
def test_greedy_matches_restatement(B, T):
    V = 40
    x = _greedy_logits(B, T, V, seed=B * 1000 + T)
    n = _lengths(B, T, seed=T)
    if B > 1:
        n[B - 1] = 0                                   # an empty utterance
    lp, tok = ops.ctc_frame_topk(x, B, T, V, n, 1)
    ids, nout, sc = ops.ctc_greedy(lp, tok, B, T, n)
    tok_c, lp_c, ids_c, n_c = tok.view(B, T).cpu(), lp.view(B, T).cpu(), ids.cpu(), n.cpu()
    for b in range(B):
        want = ctc_ref.greedy_collapse(tok_c[b], n_c[b])
        assert int(nout[b]) == len(want) and ids_c[b, :len(want)].tolist() == want, b
        assert bool((ids_c[b, len(want):] == 0).all())
        s = float(lp_c[b, :int(n_c[b])].double().sum())
        assert abs(float(sc[b]) - s) <= 1e-4 * max(1.0, abs(s))


def _check_beam(lp, tok, B, T, n, beam, label=''):
    ids, nout, sc = ops.ctc_prefix_beam(lp, tok, B, T, n, beam)
    K = tok.shape[1]
    lp_c, tok_c = lp.view(B, T, K).cpu(), tok.view(B, T, K).cpu()
    ids_c, nout_c, sc_c = ids.cpu(), nout.cpu(), sc.cpu()
    for b in range(B):
        frames = [list(zip(tok_c[b, t].tolist(), lp_c[b, t].tolist())) for t in range(int(n[b]))]
        want = ctc_ref.prefix_beam_search(frames, beam, fp32=True)
        for s in range(beam):
            if s >= len(want):
                assert int(nout_c[b, s]) == 0 and sc_c[b, s] == float('-inf'), (label, b, s)
                continue
            P, score = want[s]
            L = int(nout_c[b, s])
            assert tuple(ids_c[b, s, :L].tolist()) == P, (label, b, s)
            assert bool((ids_c[b, s, L:] == 0).all())
            assert abs(float(sc_c[b, s]) - score) <= 1e-4 * max(1.0, abs(score)), (label, b, s, float(sc_c[b, s]), score)
    return ids, nout, sc


@pytest.mark.parametrize('V', [40, 4234])
@pytest.mark.parametrize('T', [7, 249])
@pytest.mark.parametrize('beam', [1, 5, 10, 16])
def test_prefix_beam_matches_restatement(beam, T, V):
    """Every n-best token sequence identical and its score within 1e-4 relative, on the same fp32 top-40 log-probs."""
    B = 3
    x = _logits(B * T, V, seed=beam * 7 + T + V, scale=2.0)
    n = torch.tensor([T, max(1, T - 3), 1], dtype=torch.int32, device=DEV)
    lp, tok = ops.ctc_frame_topk(x, B, T, V, n, min(40, V))
    _check_beam(lp, tok, B, T, n, beam, f'beam {beam} T {T} V {V}')


def test_prefix_beam_merges_a_repeat_split_by_blank():
    """a, blank, a is the prefix (a, a) while a, a is (a,); one utterance is constructed so that the best prefix needs the
    blank path and the merge of a kept prefix with an extension."""
    V, T = 40, 9
    g = torch.Generator().manual_seed(5)
    x = 0.3 * torch.randn(T, 40, generator=g)
    for t, (k, v) in enumerate([(5, 5.0), (5, 4.0), (0, 5.0), (5, 5.0), (7, 3.0), (7, 3.0), (0, 2.0), (7, 3.0), (0, 4.0)]):
        x[t, k] += v
    x = x.to(DEV)
    n = torch.tensor([T], dtype=torch.int32, device=DEV)
    lp, tok = ops.ctc_frame_topk(x, 1, T, V, n, 40)
    ids, nout, _ = _check_beam(lp, tok, 1, T, n, 8)
    assert ids[0, 0, :int(nout[0, 0])].tolist() == [5, 5, 7, 7]


def test_prefix_beam_empty_utterance():
    V, T, B = 40, 5, 2
    x = _logits(B * T, V, seed=1)
    n = torch.tensor([T, 0], dtype=torch.int32, device=DEV)
    lp, tok = ops.ctc_frame_topk(x, B, T, V, n, 40)
    ids, nout, sc = _check_beam(lp, tok, B, T, n, 4)
    assert int(nout[1, 0]) == 0 and float(sc[1, 0]) == 0.0


# ------------------------------------------------------------------------------------------------ training
def _params(encoder_type, rate=0.0, V=40):
    fe = dict(input_size=80, output_size=256, in_channel=1, mid_channel=64, out_channel=128, kernel_size=[[3, 3], [3, 3]],
              stride=[2, 2], dropout=0.0, act_func_type='relu', front_end_layer_norm=False)
    if encoder_type == 'transformer':
        enc = dict(d_model=256, n_heads=4, d_ff=1024, n_blocks=2, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                   residual_dropout=rate, normalize_before=False, concat_after=False, activation='glu', relative_positional=False)
    else:
        enc = dict(d_model=256, d_ff=768, cov_kernel_size=5, n_heads=4, nblocks=2, pos_dropout=0.0, slf_attn_dropout=0.0,
                   ffn_dropout=0.0, residual_dropout=rate, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5, conv_bias=True,
                   activation='glu', positional_encoding=True, relative_positional=True)
    return {'type': 'ctc', 'frontend_type': 'conv', 'encoder_type': encoder_type, 'frontend': fe, 'encoder': enc,
            'encoder_output_size': 256, 'vocab_size': V}


def _build(params, seed=1234):
    torch.manual_seed(seed)
    model = CTCModel(params)
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if 'norm' in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif n.endswith('.bias'):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        for n, b in model.named_buffers():
            if n.endswith('running_mean'):
                b.normal_(0.0, 0.1, generator=g)
            elif n.endswith('running_var'):
                b.uniform_(0.8, 1.2, generator=g)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    return model.to(DEV), sd


def _batch(B=3, T=200, L=10, lens=(200, 160, 181), V=40, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, 80, generator=g)
    lens = torch.tensor(lens)
    mask = torch.arange(T)[None] < lens[:, None]
    x = x * mask.unsqueeze(2)
    tgt = torch.randint(2, V, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, L - 3:] = torch.tensor([1, 0, 0])
    tgt[1, L - 1] = 1
    tgt[2, L // 2:] = torch.tensor([1] + [0] * (L - L // 2 - 1))
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1)


def _replay(model, B, T2, p, seed):
    """The product's mask of every encoder dropout site, as the restatement's drop((prefix, k), tensor)."""
    per = 3 if model.params['encoder_type'] == 'conformer' else 2
    masks = {}
    for site, part, _ in train.dropout_sites(model):
        i, k = divmod(site - train.ENC_SITE, per)
        masks[(f'encoder.blocks.{i}', k)] = ops.dropout_mask(B * T2, 256, p, seed, site).cpu().view(B, -1, 256).float()
    return lambda s, t: t * masks[s] / (1.0 - p)


@pytest.mark.parametrize('rate', [0.0, 0.1])
@pytest.mark.parametrize('encoder_type', ['transformer', 'conformer'])
def test_training_matches_restatement(encoder_type, rate):
    params = _params(encoder_type, rate)
    model, sd = _build(params)
    x, mask, tgt, tlen = _batch()
    seed = torch.tensor([777], dtype=torch.int32, device=DEV)
    T2 = ops.conv_geometry(x.shape[1], 80)[2]
    drop = _replay(model, x.shape[0], T2, rate, seed) if rate > 0 else None
    loss_ref, g_ref, stats_ref = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd, params, drop=drop)
    with torch.no_grad():
        loss, g = train.ctc_forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV), drop_seed=seed)
    names = [n for n, _ in model.named_parameters()]
    assert set(g) == {n for n in names if g_ref[n] is not None}
    # a Conformer's depthwise_conv.bias feeds BatchNorm with batch statistics: its exact gradient is zero
    zero = [n for n in g if n.endswith('depthwise_conv.bias')]
    for n in zero:
        assert float(g[n].norm()) < 1e-3 * float(g_ref[n[:-len('bias')] + 'weight'].norm())
    worst = sorted(((_rel(g[n], g_ref[n]), n) for n in g if n not in zero), reverse=True)
    print(f'{encoder_type} rate {rate}: loss gpu {float(loss):.5f} ref {float(loss_ref):.5f}; worst '
          + ', '.join(f'{n} {r:.2e}' for r, n in worst[:4]))
    assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert worst[0][0] < REL_L2_GRAD, worst[:3]
    bufs = dict(model.named_buffers())
    for n, want in stats_ref.items():
        assert _rel(bufs[n], want) < 1e-3, n


@pytest.mark.parametrize('encoder_type', ['transformer', 'conformer'])
def test_autograd_seam_and_modes(encoder_type):
    """model.train(); loss, _ = model(...); loss.backward() fills .grad; train() under no_grad and eval() give the loss."""
    params = _params(encoder_type)
    model, sd = _build(params)
    x, mask, tgt, tlen = _batch()
    inputs, targets = {'inputs': x.to(DEV), 'mask': mask.to(DEV)}, {'targets': tgt.to(DEV), 'targets_length': tlen.to(DEV)}
    model.train()
    loss, aux = model(inputs, targets)
    assert aux is None and loss.requires_grad
    (loss * 0.5).backward()
    loss_ref, g_ref, _ = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd, params)
    used = [(n, p) for n, p in model.named_parameters() if g_ref[n] is not None and not n.endswith('depthwise_conv.bias')]
    assert all(p.grad is not None for _, p in used)
    r = _rel(torch.cat([p.grad.reshape(-1) for _, p in used]), 0.5 * torch.cat([g_ref[n].reshape(-1) for n, _ in used]))
    assert r < 2e-2, r
    with torch.no_grad():
        l_nograd, _ = model(inputs, targets)
        model.eval()
        l_eval, _ = model(inputs, targets)
    assert abs(float(l_nograd) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    if encoder_type == 'transformer':          # no BatchNorm: eval() computes the same loss
        assert abs(float(l_eval) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
    assert torch.isfinite(l_eval)


@pytest.mark.parametrize('use_graph', [False, True])
@pytest.mark.parametrize('encoder_type', ['transformer', 'conformer'])
def test_fused_trainer_follows_the_oracle_step(encoder_type, use_graph):
    """Two optimizer steps over 2 accumulated micro-batches: clip + lr(3), lr(4) + Adam, as the reference trainer."""
    params = _params(encoder_type)
    model, sd = _build(params)
    model.train()
    tr = train.FusedTrainer(model, clip_grad=0.05, accum_steps=2, use_graph=use_graph)
    names = [n for n, _ in tr.params]
    w = {n: sd[n].clone() for n in names}
    m = {n: torch.zeros_like(w[n]) for n in names}
    v = {n: torch.zeros_like(w[n]) for n in names}
    stats = {}
    for opt_step in (1, 2):
        acc = None
        for micro in range(2):
            x, mask, tgt, tlen = _batch(seed=10 * opt_step + micro)
            loss = tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV), tlen.to(DEV))
            sd_now = dict(sd)
            sd_now.update({n: w[n] for n in names})
            sd_now.update(stats)
            loss_ref, g_ref, new_stats = ctc_ref.loss_and_grads_train(x, mask, tgt, tlen, sd_now, params)
            stats.update(new_stats)
            assert abs(float(loss) - float(loss_ref)) < 2e-2 * abs(float(loss_ref))
            acc = {n: g_ref[n] / 2 for n in names} if acc is None else {n: acc[n] + g_ref[n] / 2 for n in names}
        lr = ot.transformer_lr(ot.first_step_index() + opt_step - 1, 256, 12000)
        assert abs(lr - tr.lr()) < 1e-12
        ot.clip_and_adam(w, acc, m, v, opt_step, lr, 0.05)
        torch.cuda.synchronize()
        p = dict(model.named_parameters())
        num = sum(float(((p[n].detach().cpu() - w[n]) ** 2).sum()) for n in names)
        den = sum(float(((w[n] - sd[n]) ** 2).sum()) for n in names)
        print(f'{encoder_type} graph={use_graph} step {opt_step}: rel {(num / den) ** 0.5:.3e}')
        assert (num / den) ** 0.5 < 0.3


SPEECH_MICRO_LAUNCHES = {0.0: 105, 0.1: 110}


@pytest.mark.parametrize('rate', [0.0, 0.1])
def test_speech_micro_step_launches_unchanged(rate):
    """Splitting the encoder halves out of forward_backward left the SpeechToText micro-step's kernels as they were."""
    from tests.test_gpu_train import _batch as speech_batch, _build as speech_build, _params as speech_params
    params = speech_params(n_enc=1, n_dec=1)
    params['encoder']['residual_dropout'] = rate
    params['decoder']['residual_dropout'] = rate
    x, mask, tgt = (t.to(DEV) for t in speech_batch())
    model, _ = speech_build(params)
    tr_ = train.FusedTrainer(model.train(), accum_steps=2, use_graph=False)
    counts = []
    for _ in range(3):
        n0 = ops.COUNTERS['launches']
        tr_.step(x, mask, tgt)
        counts.append(ops.COUNTERS['launches'] - n0)
    assert counts[1:] == [SPEECH_MICRO_LAUNCHES[rate] + 3, SPEECH_MICRO_LAUNCHES[rate]], counts


# ------------------------------------------------------------------------------------------------ recognition
@pytest.mark.parametrize('mode,beam', [('greedy', 1), ('beam', 10)])
def test_recognize_end_to_end(mode, beam):
    """CTCRecognizer.recognize on a small model: exactly the restatement's decode of the model's own log-probs, and those
    log-probs follow the bf16-policy oracle; where no frame's best two tokens are within the bf16 noise, the 1-best is the
    oracle's as well."""
    params = _params('transformer', V=40)
    model, sd = _build(params)
    x, mask, _, _ = _batch()
    rec = CTCRecognizer(model, beam_width=beam, mode=mode, idx2unit={i: f'u{i}' for i in range(40)})
    got = rec.recognize(x.to(DEV), mask.to(DEV))
    ids, nout, _ = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    got_ids = [row[:k] for row, k in zip(ids[:, 0].tolist(), nout[:, 0].tolist())]
    assert got == rec.translate(got_ids) and len(got) == x.shape[0]
    with torch.no_grad():
        lp, n = model.inference(x.to(DEV), mask.to(DEV))
    lp_ref, n_ref = ctc_ref.log_probs(x, mask, sd, params, policy='bf16')
    assert torch.equal(n.cpu().long(), n_ref.long())
    valid = torch.arange(lp.shape[1])[None] < n_ref[:, None]
    assert _rel(lp.cpu()[valid], lp_ref[valid]) < 2e-2

    def decode(lpb, L):
        if mode == 'greedy':
            return ctc_ref.greedy_collapse(lpb.argmax(-1), L)
        frames = [ctc_ref.frame_topk(lpb[t].tolist(), 40) for t in range(int(L))]
        return list(ctc_ref.prefix_beam_search(frames, beam, fp32=True)[0][0])

    B, T2 = x.shape[0], lp.shape[1]
    lp_c = lp.cpu()
    if mode == 'beam':              # the decode's own top-40 of the model's logits, once for the batch
        with torch.no_grad():
            lp_k, tok_k = ops.ctc_frame_topk(model.logits_bf16(x.to(DEV), mask.to(DEV))[0], B, T2, 40, n, 40)
        lp_k, tok_k = lp_k.view(B, T2, -1).cpu(), tok_k.view(B, T2, -1).cpu()
    for b in range(B):
        L = int(n[b])
        top2 = lp_ref[b, :L].topk(2, dim=-1).values
        margin = float((top2[:, 0] - top2[:, 1]).min())
        if mode == 'greedy':
            own = decode(lp_c[b], L)
        else:
            fr = [list(zip(tok_k[b, t].tolist(), lp_k[b, t].tolist())) for t in range(L)]
            own = list(ctc_ref.prefix_beam_search(fr, beam, fp32=True)[0][0])
        assert got_ids[b] == own, b
        if margin > 0.05:
            assert got_ids[b] == decode(lp_ref[b], L), (b, margin)
