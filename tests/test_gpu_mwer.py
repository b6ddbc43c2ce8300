"""GPU checks of minimum word error rate training (DESIGN.md 4.11): otb_edit_distance bit for bit against the float64
restatement (tests/mwer_ref.py), otb_mwer_coeff and otb_mwer_grad against float64 on their own fp32 inputs, the decoder
pass over K hypotheses per utterance against score_bf16 and fp32 autograd, a whole MWER pass on a fixed n-best against the
oracle, FusedTrainer(mwer_nbest=4) on the graph and eager paths, and recognize.error_counts on a real n-best."""
import random

import pytest
import torch

from tests import mwer_ref as mr

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops, train
    from opentransformer_b200.recognize import SpeechToTextRecognizer, error_counts, second_pass_rows
    DEV = torch.device('cuda:0')

from oracle import speech_model as om

REL_L2_GRAD = 4e-2        # per-parameter gradient, bf16 activations / gradients vs the fp32 oracle (as tests/test_gpu_train.py)
REL_L2_GRAD_ALL = 2e-2    # all gradients concatenated
# The MWER pass against the oracle.  Its hypotheses share most of their tokens and sum_k c_k = 0, so the MWER term's
# gradients are differences between near-equal per-hypothesis terms, and the bf16 forward's error in the softmax of every
# row is amplified there; the row-sum gradients of the decoder's last layer (the last norm3.bias, the output bias, the
# cross-attention query biases) are the most exposed.  Measured on an H100 (B 3, K 4): all gradients 1.1e-2 .. 2.6e-2,
# per tensor up to 6.4e-2, the last norm3.bias up to 1.8e-1 -- also against the oracle whose P is taken from the product's
# own l, so the excess is not in P.
REL_L2_MWER_ALL = 3e-2
REL_L2_MWER = 8e-2
REL_L2_MWER_LAST_NORM_BIAS = 2.5e-1
EOS = 1


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------------------ otb_edit_distance
def _pairs(kind, rng):
    """-> (hypotheses [N] lists, references [ceil(N / K)] lists, K)."""
    tok = lambda n, lo=2, hi=9: [rng.randint(lo, hi) for _ in range(n)]     # noqa: E731
    if kind == 'random':
        K = 3
        refs = [tok(rng.randint(0, 40)) for _ in range(20)]
        hyps = [tok(rng.randint(0, 40)) for _ in range(60)]
    elif kind == 'empty':
        K = 2
        refs = [[], [], tok(5), tok(33)]
        hyps = [[], tok(7), [], tok(32), [], [], tok(1), []]
    elif kind == 'equal_disjoint':
        K = 2
        refs = [tok(20), tok(64), tok(9, 2, 5)]
        hyps = [list(refs[0]), tok(20, 10, 20), list(refs[1]), tok(70, 10, 20), list(refs[2]), tok(9, 6, 9)]
    elif kind == 'repeats':
        K = 4
        refs = [[7] * 40, [3] * 33]
        hyps = [[7] * 40, [7] * 7, [7] * 95, [8] * 40, [3] * 32, [3] * 64, [3, 4] * 16, []]
    elif kind == 'warp_lengths':
        K = 1
        lens = [31, 32, 33, 64, 65, 255, 1023]
        refs = [tok(n, 2, 4) for n in lens] + [tok(n, 2, 4) for n in reversed(lens)]
        hyps = [tok(n, 2, 4) for n in lens] + [tok(n, 2, 4) for n in lens]
    else:       # ragged: K = 5 hypotheses of every length per utterance; N not a multiple of K
        K = 5
        refs = [tok(rng.randint(0, 70)) for _ in range(7)]
        hyps = [tok(rng.randint(0, 70)) for _ in range(33)]
    return hyps, refs, K


def _pack(rows, width=None):
    width = max([len(r) for r in rows] + [1]) if width is None else width
    out = torch.full((len(rows), width), -7, dtype=torch.int32)
    for i, r in enumerate(rows):
        out[i, :len(r)] = torch.tensor(r, dtype=torch.int32)
    return out.to(DEV), torch.tensor([len(r) for r in rows], dtype=torch.int32, device=DEV)


@pytest.mark.parametrize('kind', ['random', 'empty', 'equal_disjoint', 'repeats', 'warp_lengths', 'ragged'])
def test_edit_distance_is_exact(kind):
    hyps, refs, K = _pairs(kind, random.Random(kind))
    h, hl = _pack(hyps)
    r, rl = _pack(refs)
    got = ops.edit_distance(h, hl, r, rl, K).cpu().tolist()
    want = [mr.edit_distance(y, refs[i // K]) for i, y in enumerate(hyps)]
    assert got == want
    assert ops.edit_distance(h, hl, r, rl, K).cpu().tolist() == got


def test_edit_distance_refuses_long_rows():
    h = torch.zeros(2, 1024, dtype=torch.int32, device=DEV)
    n = torch.zeros(2, dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError, match='1023'):
        ops.edit_distance(h, n, h, n, 1)
    from opentransformer_b200 import _lib
    with pytest.raises(RuntimeError, match='1023'):
        _lib.check(_lib.lib().otb_edit_distance(ops._p(h), 1024, ops._p(n), ops._p(h), 1024, ops._p(n), 2, 1, 1024, 5, ops._p(n),
                                                ops._stream()), 'otb_edit_distance')


# ------------------------------------------------------------------------------------------------ otb_mwer_coeff / grad
def _nbest_case(seed, B=4, K=6, Lp=9):
    """Rows with duplicates, a tie in W, and an utterance whose hypotheses are all one: (tgt, n, err, tok_lp) on the host."""
    g = torch.Generator().manual_seed(seed)
    rng = random.Random(seed)
    hyps = []
    for b in range(B):
        hs = [[rng.randint(2, 30) for _ in range(rng.randint(0, Lp - 1))] for _ in range(K)]
        if b == 1:
            hs[3] = list(hs[0])
            hs[5] = list(hs[2])
        if b == 2:
            hs = [list(hs[0]) for _ in range(K)]
        hyps.append(hs)
    tgt = torch.full((B, K, Lp), -1, dtype=torch.int32)
    for b in range(B):
        for k, y in enumerate(hyps[b]):
            tgt[b, k, :len(y) + 1] = torch.tensor(y + [EOS], dtype=torch.int32)
    n = torch.tensor([[len(y) for y in hs] for hs in hyps], dtype=torch.int32)
    err = torch.tensor([[rng.randint(0, 5) for _ in range(K)] for _ in range(B)], dtype=torch.int32)
    err[3] = 2                                                                  # every W equal: zero gradient
    tok = -3.0 * torch.rand(B, K, Lp, generator=g)
    tok = torch.where(tgt >= 0, tok, torch.zeros(()))
    return hyps, tgt, n, err, tok


@pytest.mark.parametrize('scale_on_device', [False, True])
def test_mwer_coeff_matches_float64(scale_on_device):
    hyps, tgt, n, err, tok = _nbest_case(1)
    B, K, _ = tgt.shape
    scale = 0.37
    if scale_on_device:
        loss, coeff = ops.mwer_coeff(tgt.to(DEV), n.to(DEV), err.to(DEV), tok.to(DEV), 0.5,
                                     torch.tensor(scale / 0.5, dtype=torch.float32, device=DEV))
    else:
        loss, coeff = ops.mwer_coeff(tgt.to(DEV), n.to(DEV), err.to(DEV), tok.to(DEV), scale)
    loss, coeff = loss.cpu().double(), coeff.cpu().double()
    for b in range(B):
        keep = mr.kept(hyps[b])
        l = torch.stack([mr.sequence_logprob(tok[b, k], int(n[b, k])) for k in range(K)])
        want_c = mr.coefficients(l, err[b].tolist(), keep, scale)
        want_l = mr.utterance_loss(l, err[b].tolist(), keep)
        assert torch.allclose(coeff[b], want_c, rtol=1e-5, atol=1e-5), (b, coeff[b], want_c)
        assert abs(float(loss[b]) - float(want_l)) <= 2e-5 * (1 + abs(float(want_l))), (b, loss[b], want_l)
        assert all(float(coeff[b, k]) == 0.0 for k in range(K) if not keep[k])
    assert float(coeff[2].abs().max()) == 0.0 and float(loss[2]) == 0.0, 'one kept hypothesis'
    assert float(coeff[3].abs().max()) == 0.0 and float(loss[3]) == 0.0, 'equal W'


def test_mwer_coeff_clamps_lengths_to_the_row():
    """A length outside [0, Lp - 1] reads nothing outside its row: it counts as Lp - 1 (or 0)."""
    _, tgt, n, err, tok = _nbest_case(2)
    Lp = tgt.shape[2]
    args = [t.to(DEV) for t in (tgt, n, err, tok)]
    inside, outside = n.clone(), n.clone()
    inside[0, 1], outside[0, 1] = Lp - 1, 10 ** 6
    inside[1, 2], outside[1, 2] = 0, -5
    want = ops.mwer_coeff(args[0], inside.to(DEV), *args[2:], 1.0)
    got = ops.mwer_coeff(args[0], outside.to(DEV), *args[2:], 1.0)
    assert all(torch.equal(a, b) for a, b in zip(got, want))


def test_mwer_grad_matches_float64():
    g = torch.Generator().manual_seed(4)
    V, ld, Lp = 4234, 4240, 7
    H = 9
    rows = H * Lp
    logits = torch.zeros(rows, ld)
    logits[:, :V] = 4.0 * torch.randn(rows, V, generator=g)
    logits[:, V:] = 1e30                                                         # padding columns must not be read
    target = torch.randint(0, V, (rows,), generator=g, dtype=torch.int32)
    target[5::4] = -1
    coeff = torch.randn(H, generator=g) * 0.1
    coeff[3] = 0.0
    lg = logits.to(DEV)
    tok = ops.token_logprob(lg, V, target.to(DEV))
    got = ops.mwer_grad(lg, V, target.to(DEV), tok, coeff.to(DEV)).cpu()
    x = logits[:, :V].double()
    p = torch.softmax(x, dim=1)
    onehot = torch.zeros_like(p)
    live = target >= 0
    onehot[live.nonzero()[:, 0], target[live].long()] = 1.0
    want = coeff.double().repeat_interleave(Lp)[:, None] * (onehot - p)
    want[~live] = 0.0
    err = (got[:, :V].double() - want).abs()
    # the bf16 rounding of the exact value, plus the fp32 error of the softmax
    assert float((err - 2 ** -8 * want.abs() - 1e-7 * coeff.abs().repeat_interleave(Lp)[:, None].double()).max()) <= 0.0
    assert float(got[:, V:].abs().max()) == 0.0
    assert float(got[~live].abs().max()) == 0.0 and float(got[3 * Lp:4 * Lp].abs().max()) == 0.0


# ------------------------------------------------------------------------------------------------ the K-sequence decoder pass
def _decoder_model():
    from tests.test_gpu_train import _build, _params
    params = _params(n_enc=1, n_dec=2, tied=False)
    model, sd = _build(params)
    return model, sd, params


def test_decoder_pass_over_k_sequences():
    """_dec_fwd with K hypotheses per utterance: the logits against score_bf16 (the inference path's layout), and the
    gradients of the decoder and of the memory against fp32 autograd of the oracle decoder over the K-tiled memory."""
    from tests.test_gpu_model import REL_L2_LOGITS
    model, sd, params = _decoder_model()
    B, K, Lp, T2, d = 3, 4, 10, 37, 256
    g = torch.Generator().manual_seed(9)
    mem = (torch.randn(B * T2, d, generator=g)).to(torch.bfloat16)
    mem_len = torch.tensor([37, 20, 5], dtype=torch.int32)
    hyp_in = torch.randint(2, 4234, (B * K, Lp), generator=g)
    hyp_in[:, 0] = 1
    dec = model.decoder
    with torch.no_grad():
        model.eval()
        want = dec.score_bf16(hyp_in.to(DEV), mem.to(DEV), mem_len.to(DEV), B, K, Lp, T2)
        model.train()
        pk = train.TrainPack(model)
        drops = [(0.0, None, train.MWER_SITE + 3 * i) for i in range(2)]
        y, last, tape = train._dec_fwd(dec, pk, hyp_in.to(DEV), mem.to(DEV), B, K, Lp, T2, mem_len.to(DEV), drops)
        logits = train.head_fwd(y, pk.wout, pk.bout, dec.ld_logits)
        V = dec.vocab_size
        # bit for bit: the same pass with K = 1 over B*K utterances on the K-tiled memory
        tiled = mem.view(B, 1, T2, d).expand(B, K, T2, d).reshape(B * K * T2, d).contiguous().to(DEV)
        y1, _, _ = train._dec_fwd(dec, pk, hyp_in.to(DEV), tiled, B * K, 1, Lp, T2, mem_len.repeat_interleave(K).to(DEV), drops)
        assert torch.equal(train.head_fwd(y1, pk.wout, pk.bout, dec.ld_logits)[:, :V], logits[:, :V])   # columns >= V are padding
        identical = torch.equal(logits[:, :V], want[:, :V])
        print(f'training decoder over K = {K} vs score_bf16: bit-identical = {identical}, rel L2 '
              f'{_rel(logits[:, :V], want[:, :V]):.2e}')
        assert _rel(logits[:, :V], want[:, :V]) <= REL_L2_LOGITS
        R = torch.zeros(B * K * Lp, dec.ld_logits)
        R[:, :V] = torch.randn(B * K * Lp, V, generator=g) * 1e-2
        gr = train.Grads()
        dmem = train._dec_bwd(dec, pk, hyp_in.to(DEV), R.to(torch.bfloat16).to(DEV), y, last, tape, mem.to(DEV), None, gr, B, K,
                              Lp, T2, mem_len.to(DEV), drops)
    leaf = {k: v.clone().requires_grad_() for k, v in sd.items() if k.startswith('decoder.')}
    memory = mem.float().view(B, T2, d).repeat_interleave(K, 0).clone().requires_grad_()
    mmask = (torch.arange(T2)[None] < mem_len[:, None]).repeat_interleave(K, 0)
    out = om.transformer_decoder(hyp_in, memory, mmask, leaf, 'decoder.', **om.decoder_kwargs(params))
    (out.reshape(B * K * Lp, -1) * R[:, :V].to(torch.bfloat16).float()).sum().backward()
    names = [n for n in leaf if leaf[n].grad is not None]
    worst = sorted(((_rel(gr[n], leaf[n].grad), n) for n in names), reverse=True)
    r_all = _rel(torch.cat([gr[n].reshape(-1).cpu() for n in names]), torch.cat([leaf[n].grad.reshape(-1) for n in names]))
    dm_want = memory.grad.view(B, K, T2, d).sum(1).reshape(B * T2, d)
    print(f'K-sequence decoder backward: all {r_all:.2e}, dmem {_rel(dmem, dm_want):.2e}, worst ' +
          ', '.join(f'{n} {r:.2e}' for r, n in worst[:3]))
    assert r_all < REL_L2_GRAD_ALL and worst[0][0] < REL_L2_GRAD, worst[:3]
    assert _rel(dmem, dm_want) < REL_L2_GRAD


# ------------------------------------------------------------------------------------------------ the whole MWER pass
def _fixed_nbest(tgt, K, seed):
    """First-pass ids [B, K, 6] close enough in log-probability for the softmax over the n-best to spread: hypothesis k is
    the first 5 tokens of the transcript with k random substitutions, then <S/E>; utterance 0's last hypothesis repeats
    its first (a duplicate), and one row reaches the width without <S/E>."""
    g = torch.Generator().manual_seed(seed)
    B, W = tgt.shape[0], 6
    ids = torch.full((B, K, W), EOS, dtype=torch.int64)
    for b in range(B):
        for k in range(K):
            y = tgt[b, 1:6].clone()
            for _ in range(k):
                y[int(torch.randint(0, 5, (1,), generator=g))] = int(torch.randint(3, 4234, (1,), generator=g))
            ids[b, k, :5] = y
    ids[1, 2, 5] = 77
    ids[0, K - 1] = ids[0, 0]
    return ids


def _oracle_mwer(x, mask, tgt, tlen, sd, params, hyp_in, hyps, K, lam, conformer, drop=None, mwer_drop=None, coeff=None):
    """-> (loss, gradients) of the fp32 oracle with the MWER term in float64.  coeff (float64 [B, K], optional): dL/dl_k
    taken as given, so the MWER term contributes sum_k coeff_k dl_k / dtheta: the oracle's gradient with P and the
    coefficients held at coeff (the returned loss is then not the MWER loss)."""
    from tests import conformer_train_ref as cref
    leaf = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point and 'running_' not in k) for k, v in sd.items()}
    tied = params['decoder'].get('share_embedding', False)
    if tied:
        leaf['decoder.output_layer.weight'] = leaf['decoder.embedding.weight']
    stats = {}
    if conformer:
        with cref.train_mode(stats, drop):
            memory, mmask = om.encode(x, mask, leaf, params)
    else:
        om.set_dropout(drop)
        try:
            memory, mmask = om.encode(x, mask, leaf, params)
        finally:
            om.set_dropout(None)
    kw = om.decoder_kwargs(params)
    om.set_dropout(drop)
    try:
        logits = om.transformer_decoder(tgt[:, :-1], memory, mmask, leaf, 'decoder.', **kw)
    finally:
        om.set_dropout(None)
    ce = om.label_smoothing_loss(logits, tgt[:, 1:], params.get('smoothing', 0.1))
    w = params.get('ctc_weight', 0.0)
    if w > 0:
        ce = (1 - w) * ce + w * om.ctc_loss(memory, mmask, tgt[:, 1:], tlen, leaf)
    om.set_dropout(mwer_drop)
    try:
        hl = om.transformer_decoder(hyp_in, memory.repeat_interleave(K, 0), mmask.repeat_interleave(K, 0), leaf, 'decoder.', **kw)
    finally:
        om.set_dropout(None)
    B, Lp = x.shape[0], hyp_in.shape[1]
    lp = torch.log_softmax(hl.double(), dim=-1).view(B, K, Lp, -1)
    tok = torch.zeros(B, K, Lp, dtype=torch.float64)
    for b in range(B):
        for k, y in enumerate(hyps[b]):
            t = torch.tensor(y + [EOS])
            tok[b, k, :len(t)] = lp[b, k, torch.arange(len(t)), t]
    refs = [mr.reference(tgt[b], tlen[b]) for b in range(B)]
    mwer = mr.batch_loss(tok, hyps, refs) if coeff is None else (coeff * tok.sum(dim=2)).sum()
    loss = mwer + lam * ce.double()
    loss.backward()
    grads = {k: v.grad for k, v in leaf.items() if v.requires_grad and not (tied and k == 'decoder.output_layer.weight')}
    return float(loss), grads


def _product_token_logprobs(model, x, mask, seed, hyp_in, hyp_tgt, B, K, Lp):
    """The token log-probs f32 [B, K, Lp] of the n-best that forward_backward's MWER branch forms: the same training-mode
    encoder pass, the decoder over the K hypotheses with the MWER dropout sites, the head and otb_token_logprob."""
    with torch.no_grad():
        pk = train.TrainPack(model)
        mem, tr = train._encoder_fwd(model, pk, x, mask, seed)
        drops = [(r, seed, train.MWER_SITE + 3 * i) for i, r in enumerate(pk.rates['decoder'])]
        y, _, _ = train._dec_fwd(model.decoder, pk, hyp_in, mem, B, K, Lp, tr.T2, tr.lengths, drops)
        logits = train.head_fwd(y, pk.wout, pk.bout, model.decoder.ld_logits)
        tok = ops.token_logprob(logits, model.decoder.vocab_size, hyp_tgt.reshape(-1).to(torch.int32).contiguous())
    return tok.view(B, K, Lp).cpu()


@pytest.mark.parametrize('kind', ['joint_ctc', 'conformer', 'dropout'])
def test_mwer_pass_matches_oracle(kind):
    """forward_backward with a fixed n-best (duplicates, a row that reached the width without <S/E>): the loss
    mean_b L_MWER,b + lambda L_CE and every parameter gradient against the fp32 oracle with float64 MWER terms; with dropout,
    the oracle replays the product's masks at the cross-entropy sites and at the MWER branch's own sites.  Then again
    against the oracle with P taken from the product's own sequence log-probs, which leaves out the bf16 error that the
    softmax over the n-best carries into the coefficients: every tensor within 4e-2."""
    from tests.test_gpu_train import _batch
    conformer = kind == 'conformer'
    if conformer:
        from tests.test_gpu_conformer_train import _build, _params
        params = _params()
    else:
        from tests.test_gpu_train import _build, _params
        params = _params(n_enc=2, n_dec=2)
        if kind == 'joint_ctc':
            params['ctc_weight'] = 0.3
            params['encoder_output_size'] = 256
        else:
            for part in ('encoder', 'decoder'):
                params[part]['residual_dropout'] = 0.1
    model, sd = _build(params)
    if kind == 'joint_ctc':
        for k, v in model.assistor.state_dict().items():
            sd[f'assistor.{k}'] = v.detach().clone().float().cpu()
    x, mask, tgt = _batch()
    tlen = (tgt[:, 1:] != 0).sum(1).to(torch.int32)
    B, K, lam = x.shape[0], 4, 0.3
    ids = _fixed_nbest(tgt, K, seed=3)
    hyp_in, hyp_tgt, _, Lp = second_pass_rows(ids.to(DEV))
    hyps = [[mr.cut(ids[b, k]) for k in range(K)] for b in range(B)]
    assert not all(mr.kept(hyps[0])), 'the fixture must hold a duplicate'
    seed = torch.tensor([777], dtype=torch.int32, device=DEV)
    drop = mwer_drop = None
    if kind == 'dropout':
        T2, L, p = ops.conv_geometry(x.shape[1], 80)[2], tgt.shape[1] - 1, 0.1
        masks, mmasks = {}, {}
        for site, part, _ in train.dropout_sites(model):
            rows = B * T2 if part == 'encoder' else B * L
            i = (site - train.ENC_SITE) // 2 if part == 'encoder' else (site - train.DEC_SITE) // 3
            k = (site - train.ENC_SITE) % 2 if part == 'encoder' else (site - train.DEC_SITE) % 3
            masks[(f'{part}.blocks.{i}', k)] = ops.dropout_mask(rows, 256, p, seed, site).cpu().view(B, -1, 256).float()
            if part == 'decoder':
                msite = train.MWER_SITE + site - train.DEC_SITE
                mmasks[(f'decoder.blocks.{i}', k)] = ops.dropout_mask(B * K * Lp, 256, p, seed, msite).cpu().view(B * K, Lp,
                                                                                                                  256).float()
        drop = lambda site, t: t * masks[site] / (1.0 - p)          # noqa: E731
        mwer_drop = lambda site, t: t * mmasks[site] / (1.0 - p)    # noqa: E731
    loss_ref, g_ref = _oracle_mwer(x, mask, tgt, tlen, sd, params, hyp_in.cpu(), hyps, K, lam, conformer, drop, mwer_drop)
    tok = _product_token_logprobs(model.train(), x.to(DEV), mask.to(DEV), seed, hyp_in, hyp_tgt, B, K, Lp).double()
    refs = [mr.reference(tgt[b], tlen[b]) for b in range(B)]
    coeff = torch.stack([mr.coefficients(tok[b].sum(dim=1), [mr.edit_distance(y, refs[b]) for y in hyps[b]], mr.kept(hyps[b]))
                         for b in range(B)]) / B
    print(f'MWER coefficients dL/dl (float64 from the product\'s l): {coeff.tolist()}')
    assert float(coeff.abs().max()) > 1e-2, 'the n-best must be close enough for the MWER term to carry a gradient'
    _, g_same = _oracle_mwer(x, mask, tgt, tlen, sd, params, hyp_in.cpu(), hyps, K, lam, conformer, drop, mwer_drop, coeff)
    with torch.no_grad():
        loss, g = train.forward_backward(model.train(), x.to(DEV), mask.to(DEV), tgt.to(DEV), truth_length=tlen.to(DEV),
                                         drop_seed=seed, nbest=(hyp_in, hyp_tgt.view(B * K, Lp), K), mwer_ce_weight=lam)
    names = [n for n in g_ref if g_ref[n] is not None]
    # depthwise_conv.bias feeds training-mode BatchNorm, which removes any per-channel constant: its exact gradient is zero,
    # so both sides hold rounding noise (the bound of tests/test_gpu_conformer_train.py)
    for n in [n for n in names if n.endswith('depthwise_conv.bias')]:
        assert float(g[n].norm()) / float(g_ref[n[:-len('bias')] + 'weight'].norm()) < 1e-3, n
        names.remove(n)
    last_bias = f'decoder.blocks.{params["decoder"]["n_blocks"] - 1}.norm3.bias'

    def scaled(gr, n):
        return _rel(g[n], gr[n]) * (REL_L2_MWER / REL_L2_MWER_LAST_NORM_BIAS if n == last_bias else 1.0)
    worst = sorted(((scaled(g_ref, n), n) for n in names), reverse=True)
    r_all = _rel(torch.cat([g[n].reshape(-1).cpu() for n in names]), torch.cat([g_ref[n].reshape(-1) for n in names]))
    print(f'MWER pass ({kind}): loss gpu {float(loss):.5f} oracle {loss_ref:.5f}; all grads rel_l2 {r_all:.3e}; worst '
          f'(last norm3.bias scaled by {REL_L2_MWER / REL_L2_MWER_LAST_NORM_BIAS}) ' +
          ', '.join(f'{n} {r:.2e}' for r, n in worst[:3]))
    same = sorted(((scaled(g_same, n), n) for n in names), reverse=True)
    r_same = _rel(torch.cat([g[n].reshape(-1).cpu() for n in names]), torch.cat([g_same[n].reshape(-1) for n in names]))
    print(f'  with P from the product\'s l: all grads rel_l2 {r_same:.3e}; worst ' + ', '.join(f'{n} {r:.2e}' for r, n in same[:3]))
    assert abs(float(loss) - loss_ref) < 2e-2 * abs(loss_ref)
    assert r_all < REL_L2_MWER_ALL and worst[0][0] < REL_L2_MWER, worst[:3]
    assert r_same < REL_L2_MWER_ALL and same[0][0] < REL_L2_MWER, same[:3]


def test_micro_step_without_nbest_launches_unchanged():
    """mwer_nbest = 0 (the default) and a trainer that never sees an n-best launch the parent's kernels."""
    from tests.test_gpu_ctc_model import SPEECH_MICRO_LAUNCHES
    from tests.test_gpu_train import _batch, _build, _params
    params = _params(n_enc=1, n_dec=1)
    x, mask, tgt = (t.to(DEV) for t in _batch())
    model, _ = _build(params)
    tr = train.FusedTrainer(model.train(), accum_steps=2, use_graph=False, mwer_nbest=0)
    counts = []
    for _ in range(3):
        n0 = ops.COUNTERS['launches']
        tr.step(x, mask, tgt)
        counts.append(ops.COUNTERS['launches'] - n0)
    assert counts[1:] == [SPEECH_MICRO_LAUNCHES[0.0] + 3, SPEECH_MICRO_LAUNCHES[0.0]], counts


def test_fused_trainer_mwer_graph_equals_eager():
    """Two optimizer steps of FusedTrainer(mwer_nbest=4), one micro-batch each, on the CUDA-graph path and eagerly: the
    same n-best is decoded, so the losses are identical.  The weights agree to the order of the fp32 atomics that add the
    embedding gradient (an n-best repeats tokens): all but a few elements are bit-identical, and those differ by far less
    than one Adam step (lr(3) = 1.4e-7 here)."""
    from tests.test_gpu_train import _batch, _build, _params
    params = _params(n_enc=1, n_dec=1)
    x, mask, tgt = (t.to(DEV) for t in _batch())
    runs = []
    for use_graph in (False, True):
        model, _ = _build(params)
        tr = train.FusedTrainer(model.train(), clip_grad=0.05, use_graph=use_graph, mwer_nbest=4, mwer_max_len=12)
        tr.graph_after = 1
        losses = [float(tr.step(x, mask, tgt)) for _ in range(2)]
        assert model.training
        runs.append((losses, tr.flat_p.clone(), len(tr._graphs)))
    print('MWER FusedTrainer losses: eager', runs[0][0], 'graph', runs[1][0], 'graphs', runs[1][2])
    assert runs[1][2] >= 1, 'the graph path must have replayed a graph'
    assert runs[0][0] == runs[1][0]
    differ = int((runs[0][1] != runs[1][1]).sum())
    print(f'weights eager vs graph: {differ} of {runs[0][1].numel()} differ, by at most '
          f'{float((runs[0][1] - runs[1][1]).abs().max()):.3e}')
    assert differ <= 1e-3 * runs[0][1].numel()
    assert float((runs[0][1] - runs[1][1]).abs().max()) <= 5e-8          # measured 1.5e-8 on an H100


def test_trainer_keeps_one_decoder_over_ragged_batches():
    """Ragged batches bring a new frame count almost every step: the MWER trainer's recognizer keeps one BeamDecoder (with
    its KV caches and the weights it last decoded with), not one per frame count.  A recognizer's
    own max_decoders keeps the least recently used out."""
    from tests.test_gpu_train import _batch, _build, _params
    model, _ = _build(_params(n_enc=1, n_dec=1))
    tr = train.FusedTrainer(model.train(), use_graph=False, mwer_nbest=2, mwer_max_len=8)
    used = []
    for i, T in enumerate((200, 170, 150, 130, 200, 170, 150, 130)):
        x, mask, tgt = _batch(T=T, lens=(T, T - 20, T - 9), seed=i)
        tr.step(x.to(DEV), mask.to(DEV), tgt.to(DEV))
        assert len(tr._recognizer._decoders) == 1
        torch.cuda.synchronize()
        used.append(torch.cuda.memory_allocated())
    print('allocated after each step (MB):', [round(u / 2 ** 20) for u in used])
    rec = SpeechToTextRecognizer(model, beam_width=2, nbest=2, max_len=8, max_decoders=2)
    for T in (200, 170, 200, 150):
        x, mask, _ = _batch(T=T, lens=(T, T - 20, T - 9))
        rec.recognize_ids(x.to(DEV), mask.to(DEV))
    T2 = [k[2] for k in rec._decoders]
    assert T2 == [ops.conv_geometry(200, 80)[2], ops.conv_geometry(150, 80)[2]], T2


def test_error_counts_on_a_real_nbest():
    from tests.test_gpu_rescore import _inputs, _speech_model
    model, _, _ = _speech_model(eos_bias=2.0)
    B, K = 3, 5
    x, mask = _inputs(B, 200, [200, 150, 97], seed=4)
    g = torch.Generator().manual_seed(2)
    tgt = torch.zeros(B, 9, dtype=torch.int64)
    tlen = torch.tensor([8, 3, 1], dtype=torch.int32)
    for b in range(B):
        tgt[b, 0] = 1
        tgt[b, 1:tlen[b]] = torch.randint(2, 40, (int(tlen[b]) - 1,), generator=g)
        tgt[b, tlen[b]] = EOS
    rec = SpeechToTextRecognizer(model, beam_width=K, nbest=K, max_len=12)
    ids, _, _ = rec.recognize_ids(x, mask)
    got = [int(v) for v in error_counts(ids, None, tgt.to(DEV), tlen.to(DEV))]
    want = [0, 0, 0]
    for b in range(B):
        e1, emin, n = mr.error_counts([mr.cut(r) for r in ids[b].cpu()], mr.reference(tgt[b], tlen[b]))
        want = [want[0] + e1, want[1] + emin, want[2] + n]
    print('error_counts', got, 'restatement', want)
    assert got == want
    lengths = torch.full((B, K), 4, dtype=torch.int32, device=DEV)          # a CTC-style n-best: rows end at their lengths
    got = [int(v) for v in error_counts(ids, lengths, tgt.to(DEV), tlen.to(DEV))]
    want = [0, 0, 0]
    for b in range(B):
        e1, emin, n = mr.error_counts([mr.cut(r, 4) for r in ids[b].cpu()], mr.reference(tgt[b], tlen[b]))
        want = [want[0] + e1, want[1] + emin, want[2] + n]
    assert got == want
