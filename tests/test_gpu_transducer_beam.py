"""The transducer's ALSD beam search on the GPU: otb_rnnt_beam_step against one step of the float64 restatement
(tests/rnnt_beam_ref.py) on crafted search states, the carry kernels bit for bit, the whole search in lockstep with the
restatement over the GPU's own joint log-probs (eager and graph alike), the alignment sum where nothing is pruned, and
recognize's (preds, scores)."""

import numpy as np
import pytest
import torch

from opentransformer_b200 import ops, train
from opentransformer_b200.recognize import TransducerRecognizer
from tests import rnnt_beam_ref as ref
from tests.test_gpu_transducer import _batch, _build, _tie_free_model
from tests.test_rnnt_beam_ref import _lattice_score
from tests.test_rnnt_ref import params

pytestmark = pytest.mark.gpu
DEV = 'cuda'
CANARY = -7


def _f32(x):
    return float(np.float32(x))


def _rounded(utt):
    """utt with its scores rounded to fp32, the kernel's storage."""
    utt.slots = [None if s is None else (_f32(s[0]),) + s[1:] for s in utt.slots]
    utt.finals = [(_f32(f[0]),) + f[1:] for f in utt.finals]
    return utt


def _advance(lp, T, K, W, max_len, n):
    utt = ref.Utterance(K, T)
    while utt.steps < n and not utt.done:
        ref.step(utt, {j: lp(0, s[2], utt.labels(s[3])) for j, s in enumerate(utt.slots) if s is not None}, W, max_len)
        _rounded(utt)
    return utt


def _topk(row, k1):
    order = sorted(range(len(row)), key=lambda i: (-row[i], i))[:k1]
    return [row[i] for i in order], order


def _run_step(utts, rows, K, W, V, T, max_len):
    """One otb_rnnt_beam_step over the utterances utts (ref.Utterance, T frames padded) with the fp32 log-prob rows
    rows[(b, j)] of their live slots; then ref.step on each, and every output compared.  Unread inputs (padding, empty slots'
    rows) are NaN and unwritten outputs carry canaries that must survive."""
    B = len(utts)
    BK, k1, ld = B * K, min(K + 1, V), V + 3
    n_cap = K * (T + max_len) + 1
    f32 = dict(dtype=torch.float32)
    logp = torch.full((BK, ld), float('nan'), **f32)
    val = torch.full((BK, k1), float('nan'), **f32)
    idx = torch.full((BK, k1), CANARY, dtype=torch.int32)
    for (b, j), row in rows.items():
        logp[b * K + j, :V] = torch.tensor(row, **f32)
        v, i = _topk(row, k1)
        val[b * K + j] = torch.tensor(v, **f32)
        idx[b * K + j] = torch.tensor(i, dtype=torch.int32)
    st = dict(score=torch.full((BK,), float('-inf'), **f32), u=torch.zeros(BK, dtype=torch.int32),
              frame=torch.zeros(BK, dtype=torch.int32), node=torch.zeros(BK, dtype=torch.int32),
              par=torch.full((BK,), CANARY, dtype=torch.int32), tok=torch.full((BK,), CANARY, dtype=torch.long),
              node_par=torch.full((B, n_cap), CANARY, dtype=torch.int32), node_tok=torch.full((B, n_cap), CANARY, dtype=torch.int32),
              n_nodes=torch.zeros(B, dtype=torch.int32), f_score=torch.full((B, W), float('nan'), **f32),
              f_node=torch.full((B, W), CANARY, dtype=torch.int32), f_u=torch.full((B, W), CANARY, dtype=torch.int32),
              f_n=torch.zeros(B, dtype=torch.int32), done=torch.zeros(B, dtype=torch.int32),
              active=torch.tensor([sum(not u.done for u in utts) + 5], dtype=torch.int32))
    t_len = torch.tensor([u.T for u in utts], dtype=torch.int32)
    for b, utt in enumerate(utts):
        for j, s in enumerate(utt.slots):
            if s is not None:
                st['score'][b * K + j] = s[0]
                st['u'][b * K + j], st['frame'][b * K + j], st['node'][b * K + j] = s[1], s[2], s[3]
        for n, (p, t) in enumerate(utt.nodes):
            st['node_par'][b, n], st['node_tok'][b, n] = p, t
        st['n_nodes'][b] = len(utt.nodes)
        for w, f in enumerate(utt.finals):
            st['f_score'][b, w], st['f_node'][b, w], st['f_u'][b, w] = f[0], f[3], f[4]
        st['f_n'][b] = len(utt.finals)
        st['done'][b] = utt.done
    out = (torch.full((B, W, max_len), CANARY, dtype=torch.int32), torch.full((B, W), CANARY, dtype=torch.int32),
           torch.full((B, W), float('nan'), **f32))
    dst = {k: v.to(DEV) for k, v in st.items()}
    dout = tuple(t.to(DEV) for t in out)
    ops.rnnt_beam_step(logp.to(DEV), val.to(DEV), idx.to(DEV), V, T, t_len.to(DEV), dst, dout)
    got = {k: v.cpu() for k, v in dst.items()}
    ids, lengths, scores = (t.cpu() for t in dout)
    ended = 0
    for b, utt in enumerate(utts):
        was_done = utt.done
        lp = {j: np.asarray(rows[(b, j)], dtype=np.float64) for j, s in enumerate(utt.slots) if s is not None}
        par, tok = ref.step(utt, lp, W, max_len)
        sl = slice(b * K, b * K + K)
        assert got['par'][sl].tolist() == par and got['tok'][sl].tolist() == tok, b
        for j, s in enumerate(utt.slots):
            r = b * K + j
            if s is None:
                assert was_done or float(got['score'][r]) == float('-inf')
                continue
            assert abs(float(got['score'][r]) - s[0]) <= 1e-6 * max(1.0, abs(s[0])), (b, j)
            assert [int(got['u'][r]), int(got['frame'][r]), int(got['node'][r])] == list(s[1:]), (b, j)
        nn = len(utt.nodes)
        assert int(got['n_nodes'][b]) == nn
        assert got['node_par'][b, 1:nn].tolist() == [p for p, _ in utt.nodes[1:]]
        assert got['node_tok'][b, 1:nn].tolist() == [t for _, t in utt.nodes[1:]]
        assert bool((got['node_par'][b, nn:] == CANARY).all() and (got['node_tok'][b, nn:] == CANARY).all())
        nf = len(utt.finals)
        assert int(got['f_n'][b]) == nf
        for w, f in enumerate(utt.finals):
            assert abs(float(got['f_score'][b, w]) - f[0]) <= 1e-6 * max(1.0, abs(f[0]))
            assert (int(got['f_node'][b, w]), int(got['f_u'][b, w])) == (f[3], f[4])
        assert bool(got['f_score'][b, nf:].isnan().all() and (got['f_node'][b, nf:] == CANARY).all())
        assert int(got['done'][b]) == utt.done
        if utt.done and not was_done:
            ended += 1
            for w, (y, s) in enumerate(utt.nbest(W)):
                assert ids[b, w, :len(y)].tolist() == list(y) and not bool(ids[b, w, len(y):].any())
                assert int(lengths[b, w]) == len(y)
                assert (s == ref.NEG and float(scores[b, w]) == s) or abs(float(scores[b, w]) - s) <= 1e-5 * max(1.0, abs(s))
        else:
            assert bool((ids[b] == CANARY).all() and (lengths[b] == CANARY).all() and scores[b].isnan().all())
    assert int(got['active']) == int(st['active']) - ended
    return ended


@pytest.mark.parametrize('K,W,V,max_len', [(1, 1, 9, 20), (4, 4, 9, 20), (15, 15, 30, 8), (15, 3, 7, 3), (6, 2, 4, 2),
                                           (8, 5, 3, 5), (5, 3, 12, 1)])
def test_beam_step_kernel_matches_restatement(K, W, V, max_len):
    """States reached by the restatement after n steps (merges, re-formed prefixes, slots at max_len, finals at the last
    frame, full and partial n-bests, ended utterances), T_b = 0 and T_b = 1 among them; V - 1 < K in some."""
    T = 7
    ended = 0
    for seed in range(6):
        lp = ref.synthetic_lp(seed * 31 + K, V, scale=1.5, blank_bias=0.5 * (seed % 3))
        lens = [T, 1, 0, 4, T - 1 - seed % 3]
        utts = [_rounded(_advance(lambda b, t, y, bb=b: lp(bb, t, y), Tb, K, W, max_len, n))
                for b, (Tb, n) in enumerate(zip(lens, [seed * 2, 0, 0, seed, 3 + seed]))]
        rows = {(b, j): [_f32(v) for v in lp(b, s[2], utt.labels(s[3]))]
                for b, utt in enumerate(utts) for j, s in enumerate(utt.slots) if s is not None}
        ended += _run_step(utts, rows, K, W, V, T, max_len)
    assert ended > 0


def test_beam_step_kernel_ties():
    """Exact score ties (dyadic log-probs): the K best in formation order, the n-best to the earlier step and lower slot."""
    K, W, V, T, max_len = 5, 5, 4, 4, 4
    vals = (-0.5, -1.0, -2.0)

    def lp(b, t, y):
        g = np.random.default_rng([b, t, len(y)] + list(y))
        return np.array([vals[i] for i in g.integers(0, 2 if b else 3, V)], dtype=np.float64)
    def dyadic(utt):            # a crafted state on a 1/64 grid: every sum of this step is exact in fp32 and fp64 alike
        q = lambda v: round(v * 64) / 64
        utt.slots = [None if s is None else (q(s[0]),) + s[1:] for s in utt.slots]
        utt.finals = sorted(((q(f[0]),) + f[1:] for f in utt.finals), key=lambda f: (-f[0], f[1], f[2]))
        return utt
    for n in range(6):
        utts = [dyadic(_advance(lambda b, t, y, bb=b: lp(bb, t, y), T, K, W, max_len, n)) for b in range(3)]
        _run_step(utts, {(b, j): list(lp(b, s[2], utt.labels(s[3]))) for b, utt in enumerate(utts)
                         for j, s in enumerate(utt.slots) if s is not None}, K, W, V, T, max_len)


def test_carry_kernels_bit_exact():
    g = torch.Generator().manual_seed(4)
    B, K, L, H, D, T = 3, 5, 2, 24, 40, 6
    BK = B * K
    h, c = torch.randn(L, BK, H, generator=g), torch.randn(L, BK, H, generator=g)
    pp, ep = torch.randn(BK, D, generator=g).to(ops.BF16), torch.randn(B * T, D, generator=g).to(ops.BF16)
    par = torch.randint(0, K, (BK,), generator=g, dtype=torch.int32)
    frame = torch.randint(0, T, (BK,), generator=g, dtype=torch.int32)
    tok = torch.randint(0, 3, (BK,), generator=g) * torch.randint(1, 50, (BK,), generator=g)
    hg, cg = torch.full((L, BK, H), float('nan'), device=DEV), torch.full((L, BK, H), float('nan'), device=DEV)
    ppg, ep_cur = (torch.full((BK, D), float('nan'), device=DEV).to(ops.BF16) for _ in range(2))
    d = lambda t: t.to(DEV)
    ops.rnnt_beam_gather(d(par), d(frame), K, d(h), d(c), d(pp), d(ep), T, hg, cg, ppg, ep_cur)
    src = torch.arange(BK) // K * K + par.long()
    assert torch.equal(hg.cpu(), h[:, src]) and torch.equal(cg.cpu(), c[:, src]) and torch.equal(ppg.cpu(), pp[src])
    assert torch.equal(ep_cur.cpu(), ep[torch.arange(BK) // K * T + frame.long()])
    hn, cn = torch.randn(L, BK, H, generator=g), torch.randn(L, BK, H, generator=g)
    ppn = torch.randn(BK, D, generator=g).to(ops.BF16)
    oh, oc, op = d(h.clone()), d(c.clone()), d(pp.clone())
    ops.rnnt_beam_commit(d(tok), hg, cg, ppg, d(hn), d(cn), d(ppn), oh, oc, op)
    lab = tok > 0
    assert 0 < int(lab.sum()) < BK
    assert torch.equal(oh.cpu(), torch.where(lab[None, :, None], hn, hg.cpu()))
    assert torch.equal(oc.cpu(), torch.where(lab[None, :, None], cn, cg.cpu()))
    assert torch.equal(op.cpu(), torch.where(lab[:, None], ppn, ppg.cpu()))


class _GpuLattice:
    """lp(b, t, y): the GPU joint's log-probs (float64 log-softmax of its fp32 logits) at frame t of utterance b after the
    labels y, the prediction network run one token at a time from BLK and the zero state."""

    def __init__(self, model, mem, B):
        self.model, self.op = model, model._pack.get()
        op = self.op
        self.T2 = mem.shape[0] // B
        self.ep = ops.linear(mem, op['enc'].w, op['enc'].b, ops.EPI_BIAS).view(B, self.T2, -1)
        self.pred, self.rows = {}, {}

    def _state(self, y):
        if y not in self.pred:
            op = self.op
            hidden = None if not y else self._state(y[:-1])[:2]
            x = ops.embedding(torch.tensor([y[-1] if y else 0], device=DEV), op['emb'])
            out, h, c, _ = train.lstm_stack_fwd(x, op['layers'], 1, 1, hidden=hidden)
            self.pred[y] = (h, c, ops.linear(out, op['dec_w']))
        return self.pred[y]

    def __call__(self, b, t, y):
        y = tuple(y)
        if (b, t, y) not in self.rows:
            hj = ops.rnnt_joint(self.ep[b, t:t + 1].contiguous(), self._state(y)[2], 1, 1, 1)
            logits = ops.linear(hj, self.op['out_w'], self.op['out_b'], ops.EPI_BIAS, out_f32=True,
                                n_out=self.model.joint.ld_logits)
            self.rows[(b, t, y)] = torch.log_softmax(logits[0, :self.model.vocab_size].double().cpu(), -1).numpy()
        return self.rows[(b, t, y)]


@pytest.mark.parametrize('K,W,max_len', [(1, 1, 1023), (4, 1, 1023), (4, 4, 1023), (15, 1, 1023), (15, 4, 1023), (1, 1, 4),
                                         (4, 4, 4), (15, 4, 4)])
def test_alsd_search_in_lockstep_with_restatement(K, W, max_len):
    x, mask, _, _ = _batch(lens=(120, 60, 97), seed=5)
    model = _tie_free_model(11, x, mask)
    res = {}
    for use_graph in (False, True):
        rec = TransducerRecognizer(model, mode='alsd', beam_width=K, nbest=W, max_len=max_len, use_graph=use_graph)
        res[use_graph] = [t.clone() for t in rec.recognize_ids(x.to(DEV), mask.to(DEV))]
    for a, b in zip(res[False], res[True]):
        assert torch.equal(a, b)
    ids, n, sc = res[True]
    assert tuple(ids.shape) == (3, W, max_len) and tuple(n.shape) == (3, W) and tuple(sc.shape) == (3, W)
    with torch.no_grad():
        mem, lengths, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        want = ref.search(_GpuLattice(model, mem, B), lengths.cpu().tolist(), K, W, max_len)
    print(K, W, max_len, [u.steps for u in want], n.tolist())
    for b, utt in enumerate(want):
        for w, (y, s) in enumerate(utt.nbest(W)):
            assert int(n[b, w]) == len(y) and ids[b, w, :len(y)].tolist() == list(y)
            assert not bool(ids[b, w, len(y):].any())
            if s == ref.NEG:
                assert float(sc[b, w]) == s
            else:
                assert abs(float(sc[b, w]) - s) <= 1e-5 * abs(s), (b, w, float(sc[b, w]), s)
    assert all(len(u.finals) > 0 for u in want)


def test_unpruned_alsd_on_gpu_sums_every_alignment():
    """V = 3 and max_len = 2: 7 label sequences, K = W = 7 keeps every prefix, so each n-best score is the lattice's sum
    over all alignments of its labels under the GPU's own log-probs."""
    x, mask, _, _ = _batch(T=40, lens=(40, 23, 31), seed=2)
    model, _ = _build(params(layers=1, V=3), seed=9)
    model.eval()
    rec = TransducerRecognizer(model, mode='alsd', beam_width=7, nbest=7, max_len=2)
    ids, n, sc = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    with torch.no_grad():
        mem, lengths, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        lat = _GpuLattice(model, mem, B)
    for b in range(B):
        seqs = set()
        for w in range(7):
            y = tuple(ids[b, w, :int(n[b, w])].tolist())
            seqs.add(y)
            want = _lattice_score(lat, b, int(lengths[b]), y)
            assert abs(float(sc[b, w]) - want) <= 1e-5 * abs(want), (b, y, float(sc[b, w]), want)
        assert len(seqs) == 7
        assert all(float(sc[b, w]) >= float(sc[b, w + 1]) for w in range(6))


def test_recognize_returns_preds_and_scores():
    x, mask, _, _ = _batch(lens=(120, 60, 97), seed=5)
    model = _tie_free_model(11, x, mask)
    rec = TransducerRecognizer(model, mode='alsd', beam_width=4, nbest=3, max_len=30)
    ids, n, sc = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    preds, scores = rec.recognize(x.to(DEV), mask.to(DEV))
    assert torch.equal(preds, ids) and torch.equal(scores, sc)
    units = {i: f'u{i}' for i in range(model.vocab_size)}
    preds, scores = TransducerRecognizer(model, idx2unit=units, mode='alsd', beam_width=4, nbest=3,
                                         max_len=30).recognize(x.to(DEV), mask.to(DEV))
    assert torch.equal(scores, sc)
    want = []
    for b in range(3):
        row = []
        for w in range(3):
            y = ids[b, w, :int(n[b, w])].tolist()
            y = y[:y.index(1)] if 1 in y else y             # nbest_translate ends a hypothesis at <S/E>
            row.append(' '.join(units[t] for t in y))
        want.append(row)
    assert preds == want
