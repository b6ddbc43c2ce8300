"""The persistent decode kernel (csrc/decode_group.cu) at the edges of the configurations BeamDecoder.mega_supported()
sends to it, step by step against a float64 decoder and the tie-exact beam step of tests/beam_ties_ref.py.

Each case builds BeamDecoder(..., persistent=True) straight from a random bf16 memory [B * T, 256] and per-utterance
memory lengths (no encoder, so T and mem_len are exact), runs the whole search in one launch with the per-step log-prob
and score traces on, and then at every step:
  * ids bit-exact: the kernel's own log-probs drive the tie-exact beam step; tokens, parents and scores must be equal;
  * log-probs close: the live rows against the oracle's full-prefix decoder_inference on float64 copies of the weights and
    of the memory (the sinusoid table stays fp32, as the kernel's), within the limits of tests/test_gpu_model.py;
  * end of search: the executed step count equals the reference loop's, and finalize is bit-exact.
Each case is built to reach one branch of the kernel's beam step (the logit rows of an utterance gathered into shared
memory or read in place; the per-row top-k from the candidate list, from a degenerate threshold or by the flat-row
fallback), and prints which one with its worst log-prob errors."""
import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import ops
    from opentransformer_b200.recognize import BeamDecoder
    DEV = torch.device('cuda:0')

from oracle import speech_model as om
from tests import beam_ties_ref as btr
from tests.test_gpu_model import MAX_ABS_FRAC, REL_L2_LOGITS, _build, _params, _rel

D = 256
STAGE_BYTES = 65536 + 2 * 65536      # shared memory the kernel gathers an utterance's logit rows into (A tile + 2 stages)
TIE_BIAS = 20.0                      # common logit of the tied token set: far above every other logit of the untied layer


def _branch(V, beam, tie):
    """Which path of the beam step a case reaches (decode_group.cu, beam_step): gathered / in place, and the top-k route."""
    ldv4 = (V + 31) // 32 * 32 // 4
    nbox = (ldv4 + 63) // 64
    gathered = nbox * 64 * (beam | 1) * 16 <= STAGE_BYTES
    if (V + 3) // 4 < beam:
        route = 'degenerate threshold'           # fewer than `beam` lanes hold a finite logit
    elif (tie == 'all' and V - 1 > 128) or (isinstance(tie, int) and tie > 128):
        route = 'flat-row fallback'              # more than 128 logits of a row are >= the lane-maxima threshold
    else:
        route = 'candidate list'
    return ('gathered' if gathered else 'in place') + ', ' + route


def _model(c):
    params = _params(n_enc=1, n_dec=c['layers'])
    untied = c['tie'] is not None or c['eos'] != -1e4
    params['decoder'].update(vocab_size=c['V'], share_embedding=not untied)
    model, _ = _build(params, seed=1234 + c['seed'])
    dec = model.decoder
    V = c['V']
    with torch.no_grad():
        ow, ob = dec.output_layer.weight, dec.output_layer.bias
        if c['tie'] == 'all':                    # all-zero output layer: every logit 0 but EOS, in every row
            ow.zero_()
            ob.zero_()
        elif c['tie'] is not None:               # S ties exactly in every row: zero weight rows and one common bias
            g = torch.Generator().manual_seed(99 + c['tie'])
            S = 2 + torch.randperm(V - 2, generator=g)[:c['tie']]       # excludes token 1 (BOS / EOS)
            lanes = torch.unique((S // 4) % 32).numel()
            assert lanes >= c['beam'], 'the tied set must cover at least `beam` lanes of the threshold scan'
            ow[S.to(DEV)] = 0.0
            ob[S.to(DEV)] = TIE_BIAS
        ob[1] = c['eos']
    sd64 = {f'decoder.{k}': v.detach().double() for k, v in dec.state_dict().items()}
    return dec, sd64, om.decoder_kwargs(params)


def _run(dec, c, mem, lens, barrier='default'):
    """One launch of the whole search with the traces on -> (BeamDecoder, dbg_logp, dbg_scores)."""
    B, beam, T, L = c['B'], c['beam'], c['T'], c['max_len']
    bd = BeamDecoder(dec, B, beam, T, L, DEV, use_graph=False, persistent=True)
    assert bd.persistent, 'this configuration is inside the envelope: it must run on the persistent kernel'
    bd.setup(mem, lens)
    dbg_logp = torch.zeros(L, B * beam, c['V'], dtype=torch.float32, device=DEV)
    dbg_scores = torch.zeros(L, B * beam, dtype=torch.float32, device=DEV)
    try:
        ops.set_decode_barrier(barrier)
        bd.run_persistent(L, dbg_logp, dbg_scores)
        torch.cuda.synchronize()
    finally:
        ops.set_decode_barrier('default')
    return bd, dbg_logp, dbg_scores


def _lockstep(c):
    dec, sd64, kw = _model(c)
    B, beam, T, L, V = c['B'], c['beam'], c['T'], c['max_len'], c['V']
    N = B * beam
    g = torch.Generator().manual_seed(500 + c['seed'])
    mem = torch.randn(B * T, D, generator=g).to(torch.bfloat16).to(DEV)
    lens = torch.tensor(c['lens'], dtype=torch.int32)
    assert lens.numel() == B and int(lens.max()) <= T and int(lens.min()) >= 1
    with torch.no_grad():
        bd, dbg_logp, dbg_scores = _run(dec, c, mem, lens.to(DEV), 'cluster' if c['barrier'] else 'default')
        steps_gpu = int(bd.state.ctrl[0].item())
        mem64 = mem.double().view(B, T, D)
        mmask = (torch.arange(T)[None] < lens[:, None]).to(DEV)
        cols = torch.tensor([v for v in range(V) if not (v == 1 and c['eos'] == -1e4)])   # EOS column: -1e4 bias
        sample = c['logp_utts']
        preds = torch.full((N, 1), 1, dtype=torch.long)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        worst, worst_rel, scale, steps_ref, checked = 0.0, 0.0, 1e-9, L, 0
        utt_end = [L] * B
        for s in range(L):
            lp_gpu = dbg_logp[s].cpu()
            utt_alive = (~flag.view(B, beam)).any(dim=1).repeat_interleave(beam)   # a group stops once all its rows ended
            alive = (~flag.view(-1)) & utt_alive
            if sample is not None:
                alive &= (torch.arange(N) // beam) % sample == 0
            if (s % c['logp_every'] == 0 or s == L - 1) and bool(alive.any()):
                rows = alive.nonzero().view(-1)
                with torch.device(DEV):
                    ref = om.decoder_inference(preds[rows].to(DEV), mem64[rows.to(DEV) // beam],
                                               mmask[rows.to(DEV) // beam], sd64, 'decoder.', **kw)
                ref = ref[:, cols.to(DEV)].cpu()
                got = lp_gpu[rows][:, cols].double()
                worst = max(worst, float((got - ref).abs().max()))
                worst_rel = max(worst_rel, _rel(got, ref))
                scale = max(scale, float(ref.abs().max()))
                checked += 1
            preds, scores, flag = btr.beam_step(lp_gpu, preds, scores, flag, beam)
            assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'token / parent ids differ at step {s}'
            assert torch.equal(dbg_scores[s].cpu(), scores.view(-1)), f'scores differ at step {s}'
            for u in range(B):
                if utt_end[u] == L and bool(flag.view(B, beam)[u].all()):
                    utt_end[u] = s + 1
            if bool(flag.all()):
                steps_ref = s + 1
                break
        assert steps_gpu == steps_ref, f'executed step count: kernel {steps_gpu} vs reference loop {steps_ref}'
        assert torch.equal(bd.state.scores.cpu(), scores.view(-1))
        for penalty in (0.0, 0.6):
            nb, ns = btr.beam_finalize(preds, scores, beam, beam, penalty, 5)
            gp, gs = bd.state.finalize(penalty, 5, beam)
            assert torch.equal(gp[:, :, :steps_ref].cpu(), nb), f'finalize ids differ (penalty {penalty})'
            if penalty == 0.0:
                assert torch.equal(gs.cpu(), ns), 'finalize scores differ'
            else:       # powf on the device against torch.pow on the host
                torch.testing.assert_close(gs.cpu(), ns, rtol=1e-6, atol=1e-6)
        if c['barrier']:     # the software group barrier changes scheduling only: every output bit-identical
            bd2, lp2, sc2 = _run(dec, c, mem, lens.to(DEV), 'software')
            for a, b in ((bd.state.tok_hist, bd2.state.tok_hist), (bd.state.par_hist, bd2.state.par_hist),
                         (bd.state.scores, bd2.state.scores), (bd.state.ctrl[:2], bd2.state.ctrl[:2]),
                         (dbg_logp, lp2), (dbg_scores, sc2)):
                assert torch.equal(a, b), 'cluster and software group barriers give different results'
    print(f"[{c['name']}] V={V} beam={beam} B={B} T={T} mem_len={c['lens'][:8]} layers={c['layers']} "
          f"max_len={L}: {_branch(V, beam, c['tie'])}; {steps_ref} steps, ids / parents / scores bit-exact; "
          f"log-probs vs float64 at {checked} steps: rel_l2<={worst_rel:.3e} max_abs={worst:.3e} (|ref|_inf {scale:.3e})")
    assert worst_rel < REL_L2_LOGITS and worst < MAX_ABS_FRAC * scale
    return steps_ref, utt_end


def _case(name, **kw):
    c = dict(name=name, V=4234, beam=4, B=2, T=32, lens=None, max_len=8, layers=1, tie=None, eos=-1e4, logp_every=1,
             logp_utts=None, barrier=False, seed=0)
    c.update(kw)
    if c['lens'] is None:
        c['lens'] = [c['T'] - (7 * u) % c['T'] for u in range(c['B'])]
    return c


def _groups_full():
    return (128 // 10) * (ops.num_sms() // 16)


CASES = [
    # memory length: one frame, and T - 1 / T / the 128-frame boundary of the cross-attention tiles
    _case('mem_T1', T=1, lens=[1, 1]),
    _case('mem_T16', T=16, B=3, lens=[1, 15, 16]),
    _case('mem_T128', T=128, B=3, lens=[1, 127, 128]),
    _case('mem_T129', T=129, B=3, lens=[1, 128, 129]),
    _case('mem_T256', T=256, B=6, lens=[1, 255, 256, 127, 128, 129]),
    # prefix: every step of a 128-step search (8-position self-attention half-buffers, the 128-entry ancestry row)
    _case('prefix_128', T=40, lens=[40, 23], max_len=128),
    # vocabulary / top-k route / gathered or in place
    _case('V16_beam16', V=16, beam=16, max_len=6),
    _case('V17_beam16', V=17, beam=16, max_len=6),
    _case('V33_beam4', V=33, B=3, max_len=6),
    _case('V4234_beam11', beam=11, B=3, max_len=6),
    _case('V4234_beam12', beam=12, B=3, max_len=6),
    _case('V9728_beam4', V=9728, B=3, max_len=6),
    _case('V9729_beam4', V=9729, B=3, max_len=6),
    # row groups with dead rows, the last group holding one utterance
    _case('groups_beam3', beam=3, B=128 // 3 + 1, T=24, max_len=5),
    _case('groups_beam7', beam=7, B=128 // 7 + 1, T=24, max_len=5),
    _case('groups_beam9', beam=9, B=128 // 9 + 1, T=24, max_len=5),
    _case('groups_beam13', beam=13, B=128 // 13 + 1, T=24, max_len=5),
    # depth
    _case('layers8', layers=8, B=3, T=64, max_len=10, barrier=True),
    # exact ties: |S| equal maxima in every row (129 and more: the flat-row fallback); all-zero output layer
    _case('tie127', tie=127, beam=4, B=3, max_len=6, barrier=True),
    _case('tie128', tie=128, beam=10, B=3, max_len=6, barrier=True),
    _case('tie129', tie=129, beam=12, B=3, max_len=6, barrier=True),
    _case('tie300', tie=300, beam=16, B=2, max_len=6, barrier=True),
    _case('tie_all_zero', tie='all', beam=8, B=3, max_len=6, barrier=True),
]


@pytest.mark.parametrize('c', CASES, ids=[c['name'] for c in CASES])
def test_persistent_envelope_lockstep(c):
    steps, _ = _lockstep(c)
    assert steps == c['max_len']          # EOS carries -1e4: every search runs to max_len


def test_persistent_full_grid_lockstep():
    """Every row group the GPU holds at 16 CTAs each, beam 10 (12 utterances, 8 dead rows per group): ids at every step,
    log-probs on every fifth utterance, under both group barriers."""
    B = _groups_full()
    c = _case('full_grid', beam=10, B=B, T=24, max_len=5, logp_utts=5, barrier=True)
    steps, _ = _lockstep(c)
    assert steps == c['max_len']


def test_persistent_early_end_in_two_row_groups():
    """EOS bias 2 on an untied output layer: hypotheses end at different steps, and utterances of the two row groups end at
    different steps; the kernel's step count and its filled-in history of the group that ended first must match."""
    beam = 13
    c = _case('early_end', beam=beam, B=12, T=48, max_len=40, eos=2.0, seed=3)
    steps, utt_end = _lockstep(c)
    upg = 128 // beam
    ends = [max(utt_end[g * upg:(g + 1) * upg]) for g in range(-(-c['B'] // upg))]
    print(f'early end: search ran {steps} of {c["max_len"]} steps; per-utterance end {utt_end}; per-group end {ends}')
    assert steps < c['max_len'] and len(set(ends)) > 1


def test_envelope_boundary():
    """mega_supported() is true at T 256, max_len 128, 8 layers and the full grid, and false one step past each limit;
    past it the search runs on the per-step graph path and finishes."""
    full = _groups_full()
    c8 = _case('boundary8', V=64, layers=8)
    c9 = _case('boundary9', V=64, layers=9)
    dec8, _, _ = _model(c8)
    dec9, _, _ = _model(c9)
    assert BeamDecoder(dec8, full, 10, 256, 128, DEV, persistent=True).persistent
    for dec, B, beam, T, L in ((dec8, 2, 4, 257, 8), (dec8, 2, 4, 40, 129), (dec9, 2, 4, 40, 8),
                               (dec8, full + 1, 10, 24, 8)):
        bd = BeamDecoder(dec, B, beam, T, L, DEV, persistent=True)
        assert not bd.mega_supported() and not bd.persistent, (B, beam, T, L, len(dec.blocks))
        g = torch.Generator().manual_seed(T)
        mem = torch.randn(B * T, D, generator=g).to(torch.bfloat16).to(DEV)
        with torch.no_grad():
            bd.setup(mem, torch.full((B,), T, dtype=torch.int32, device=DEV))
            steps = bd.run(L)
            gp, gs = bd.state.finalize(0.6, 5, 1)
        assert steps == L and gp.shape == (B, 1, L) and bool(torch.isfinite(gs).all())
