"""CPU checks of the pruned RNN-T restatement (tests/rnnt_pruned_ref.py), the transducer's prune_range configuration,
and the resources of the pruned loss's kernels (ptxas, sm_90a)."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch
import torchaudio.functional as TAF

from opentransformer_b200 import build
from opentransformer_b200 import model as M
from tests import rnnt_pruned_ref as prr
from tests import rnnt_ref
from tests.test_rnnt_ref import params


def _pruned_params(S=3, alpha=0.5, **kw):
    p = params(**kw)
    p['joint'] = dict(p['joint'], prune_range=S, simple_loss_scale=alpha)
    return p


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_simple_loss_equals_torchaudio(seed):
    g = torch.Generator().manual_seed(seed)
    B, T, U, V = 3, 7, 4, 11
    am = 2 * torch.randn(B, T, V, generator=g, dtype=torch.float64)
    lm = 2 * torch.randn(B, U + 1, V, generator=g, dtype=torch.float64)
    labels = torch.randint(1, V, (B, U), generator=g, dtype=torch.int32)
    t_len, u_len = torch.tensor([7, 3, 5], dtype=torch.int32), torch.tensor([4, 2, 0], dtype=torch.int32)
    want = TAF.rnnt_loss((am[:, :, None] + lm[:, None]).float(), labels, t_len, u_len, blank=0, reduction='none').double()
    for b in range(B):
        Tb, Ub = int(t_len[b]), int(u_len[b])
        lpb, lpy = prr.simple_logprobs(am[b, :Tb], lm[b, :Ub + 1], labels[b, :Ub].long())
        got = rnnt_ref.lattice_nll(lpb, lpy)
        assert abs(float(got) - float(want[b])) <= 1e-4 * abs(float(want[b]))


def _random_lattice(T, U, V, seed):
    g = torch.Generator().manual_seed(seed)
    logits = 2 * torch.randn(T, U + 1, V, generator=g, dtype=torch.float64)
    labels = torch.randint(1, V, (U,), generator=g)
    return rnnt_ref.node_logprobs(logits, labels)


@pytest.mark.parametrize('T,U', [(6, 4), (9, 7), (3, 2)])
def test_wide_bands_are_the_full_loss(T, U):
    lpb, lpy = _random_lattice(T, U, 9, T * 10 + U)
    for S in (U + 1, U + 3):
        s = prr.prune_ranges(prr.occupancy(lpb, lpy).float().numpy(), T, U, S)
        assert s.tolist() == [0] * T
        assert abs(float(prr.band_nll(lpb, lpy, s, S)) - float(rnnt_ref.lattice_nll(lpb, lpy))) < 1e-12


@pytest.mark.parametrize('seed', range(4))
def test_pruned_nll_bounds_the_full_nll(seed):
    T, U = 8, 6
    lpb, lpy = _random_lattice(T, U, 7, 100 + seed)
    full = float(rnnt_ref.lattice_nll(lpb, lpy))
    occ = prr.occupancy(lpb, lpy).float().numpy()
    for S in (2, 3, 4, 5, 7):
        s = prr.prune_ranges(occ, T, U, S)
        assert float(prr.band_nll(lpb, lpy, s, S)) >= full - 1e-12


def test_ranges_satisfy_the_rule_over_random_occupancies():
    rng = np.random.default_rng(5)
    for _ in range(300):
        T = int(rng.integers(1, 12))
        S = int(rng.integers(2, 6))
        U = int(rng.integers(0, T * (S - 1) + 1))
        occ = rng.random((T, U + 1)).astype(np.float32) * (rng.random((T, U + 1)) < 0.6)
        s = prr.prune_ranges(occ, T, U, S)
        assert prr.check_ranges(s, T, U, S) == [], (T, U, S, s)
        assert prr.has_complete_path(s, T, U, S), (T, U, S, s)


def test_too_long_transcript_has_no_path():
    T, S = 3, 3
    U = T * (S - 1) + 1
    lpb, lpy = _random_lattice(T, U, 6, 9)
    s = prr.prune_ranges(prr.occupancy(lpb, lpy).float().numpy(), T, U, S)
    assert not prr.has_complete_path(s, T, U, S)
    assert float(prr.band_nll(lpb, lpy, s, S)) == float('inf')


def test_argmax_takes_the_lowest_window_on_a_tie():
    occ = np.ones((3, 4), dtype=np.float32)
    assert prr.prune_ranges(occ, 3, 3, 2).tolist() == [0, 1, 2]    # every window ties at s = 0; the bands are raised to reach U


# ------------------------------------------------------------------------------------------------ configuration
def test_keys_without_prune_range_are_unchanged():
    torch.manual_seed(0)
    plain = set(M.TransducerModel(params()).state_dict())
    torch.manual_seed(0)
    none = M.TransducerModel(dict(params(), joint={'inner_size': 64, 'prune_range': None}))
    assert set(none.state_dict()) == plain
    torch.manual_seed(0)
    pruned = M.TransducerModel(_pruned_params())
    assert set(pruned.state_dict()) - plain == {'joint.simple_am_proj.weight', 'joint.simple_am_proj.bias',
                                               'joint.simple_lm_proj.weight', 'joint.simple_lm_proj.bias'}
    assert tuple(pruned.joint.simple_am_proj.weight.shape) == (40, 128)
    assert tuple(pruned.joint.simple_lm_proj.weight.shape) == (40, 64)
    assert pruned.joint.prune_range == 3 and pruned.joint.simple_loss_scale == 0.5


@pytest.mark.parametrize('bad', [1, 0, -3, 2.0, '5', True])
def test_bad_prune_range_is_refused(bad):
    p = params()
    p['joint'] = {'inner_size': 64, 'prune_range': bad}
    with pytest.raises(ValueError):
        M.TransducerModel(p)


def test_refusals_of_the_transducer_still_hold():
    p = _pruned_params()
    p['decoder_type'] = 'transformer'
    with pytest.raises(NotImplementedError):
        M.TransducerModel(p)
    p = _pruned_params()
    p['joint'] = dict(p['joint'], inner_size=60)
    with pytest.raises(NotImplementedError):
        M.TransducerModel(p)


def test_restated_objective_with_wide_bands_is_simple_plus_full():
    """With S past every transcript, the pruned term is the full lattice loss."""
    p = _pruned_params(S=20, alpha=0.25)
    torch.manual_seed(3)
    model = M.TransducerModel(p)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    B, T, L = 2, 40, 6
    x = torch.randn(B, T, 80, generator=g)
    mask = torch.ones(B, T, dtype=torch.bool)
    tgt = torch.randint(2, 40, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[1, L - 2:] = torch.tensor([1, 0])
    tlen = (tgt[:, 1:] != 0).sum(1)
    tgt[0, L - 1] = 1
    loss, _ = prr.model_loss(x, mask, tgt, tlen, sd, p)
    full, _ = rnnt_ref.model_loss(x, mask, tgt, tlen, sd, p)
    memory, mmask, _ = rnnt_ref._encode_train(x, mask, sd, p, None, 'bf16')
    labels = tgt[:, 1:-1]
    toks = torch.cat((torch.zeros(B, 1, dtype=torch.long), labels), 1)
    gp = rnnt_ref.predictor(toks, sd, 1, 'bf16')
    am = prr.om.linear(memory, sd, 'joint.simple_am_proj', 'bf16')
    lm = prr.om.linear(gp, sd, 'joint.simple_lm_proj', 'bf16')
    simple = rnnt_ref.batch_loss(am[:, :, None] + lm[:, None], labels, mmask.sum(-1), tlen - 1)
    assert abs(float(loss) - float(0.25 * simple + full)) < 1e-4 * float(loss)


# ------------------------------------------------------------------------------------------------ kernel resources
def test_pruned_kernels_compile_without_spills(tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip('nvcc is not available')
    if os.path.isabs(nvcc) and not os.path.exists(nvcc):
        pytest.skip('nvcc is not available')
    report = ''
    for src in ('rnnt.cu', 'rnnt_pruned.cu'):
        cmd = [nvcc] + build.NVCC_FLAGS + ['-c', os.path.join(build.CSRC, src), '-o', str(tmp_path / (src + '.o'))]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=str(tmp_path))
        assert r.returncode == 0, r.stdout
        report += r.stdout
    names = ['rnnt_joint_kernel', 'rnnt_joint_bwd_kernel', 'rnnt_logprob_kernel', 'rnnt_loss_kernel', 'rnnt_dlogits_kernel',
             'rnnt_simple_lse_kernel', 'rnnt_simple_bwd_kernel', 'rnnt_prune_ranges_kernel']
    for n in names:
        m = re.search(r'Function properties for _ZN3otb\d+' + n + r'\S*\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, '
                      r'(\d+) bytes spill loads', report)
        assert m, f'no ptxas report for {n}'
        assert tuple(int(x) for x in m.groups()) == (0, 0, 0), (n, m.groups())
