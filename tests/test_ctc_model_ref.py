"""CPU checks of the CTC-only model: the CPU restatement (tests/ctc_ref.py) against the reference's own CTCModel in train()
and its greedy collapse (tests/golden/live_ref_ctc.pt), the prefix beam search against every alignment enumerated, the
registry, key names, checkpoint round trip and recogniser factory, and the refusals, which come before any device work."""
import copy
import math
import os
from types import SimpleNamespace

import pytest
import torch

from tests import ctc_ref
from tests.test_head_dim_96 import CONFORMER_BASELINE, synth_state_dict
from tests.test_transformer_lm_ref import sample

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'live_ref_ctc.pt')


@pytest.fixture(scope='module')
def fixture():
    return torch.load(GOLDEN, weights_only=False)


@pytest.mark.parametrize('encoder_type', ['transformer', 'conformer'])
def test_restatement_equals_live_reference_in_train_mode(fixture, encoder_type):
    """Loss, every parameter gradient (a Conformer's post_ffn.* gets none) and the BatchNorm running statistics of
    End2EndModel['ctc'] in train() on a ragged batch: the targets are truth[:, 1:-1] with targets_length - 1 labels."""
    c = fixture['train'][encoder_type]
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    loss, grads, stats = ctc_ref.loss_and_grads_train(c['x'], c['mask'], c['tgt'], c['tlen'], sd, c['params'])
    torch.testing.assert_close(loss, c['loss_ref'], rtol=1e-5, atol=1e-5)
    g_ref = c['g_ref']
    assert set(grads) == set(g_ref), set(grads) ^ set(g_ref)
    for n, want in g_ref.items():
        if want is None:
            assert grads[n] is None and '.post_ffn.' in n, n
            continue
        torch.testing.assert_close(sample(grads[n]), want, rtol=1e-4, atol=1e-6, msg=lambda m, n=n: f'{n}: {m}')
    assert set(stats) == {n for n in c['stats_ref'] if 'running_' in n}
    for n, want in c['stats_ref'].items():
        if 'num_batches' in n:
            assert int(want) == 1
            continue
        torch.testing.assert_close(stats[n], want, rtol=1e-5, atol=1e-6, msg=lambda m, n=n: f'{n}: {m}')


def test_joint_ctc_would_keep_the_eos():
    """The CTC-only targets differ from joint CTC's (truth[:, 1:], targets_length): dropping <S/E> changes the loss."""
    c = torch.load(GOLDEN, weights_only=False)['train']['transformer']
    sd = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    from oracle import speech_model as om
    memory, mmask = om.encode(c['x'], c['mask'], sd, c['params'])
    joint = om.ctc_loss(memory, mmask, c['tgt'][:, 1:], c['tlen'], sd)
    assert abs(float(joint) - float(c['loss_ref'])) > 1e-3


def test_greedy_collapse_equals_reference(fixture):
    g = fixture['greedy']
    best = g['lp'].argmax(-1)
    got = [ctc_ref.greedy_collapse(best[b], g['lengths'][b]) for b in range(best.shape[0])]
    assert got == g['ids_ref']
    assert [] in got and any(len(x) == 1 for x in got)


@pytest.mark.parametrize('T,V,seed', [(6, 4, 0), (6, 4, 1), (5, 3, 2), (4, 5, 3), (1, 4, 4)])
def test_prefix_beam_without_pruning_is_exact(T, V, seed):
    """With K >= V and a beam larger than the number of distinct prefixes nothing is pruned: the search then returns every
    prefix with its exact marginal over all alignments, which enumeration gives in fp64."""
    lp = torch.log_softmax(ctc_ref.synth_log_probs(T, V, seed).double(), dim=-1)
    want = ctc_ref.prefix_marginals(lp.tolist())
    frames = [ctc_ref.frame_topk(lp[t].tolist(), V) for t in range(T)]
    got = ctc_ref.prefix_beam_search(frames, beam=10 ** 6)
    assert {p for p, _ in got} == set(want)
    for p, s in got:
        assert abs(s - want[p]) < 1e-9, (p, s, want[p])
    assert [s for _, s in got] == sorted((s for _, s in got), reverse=True)
    assert abs(math.log(sum(math.exp(s) for _, s in got))) < 1e-9          # the prefixes partition every alignment


def test_prefix_beam_merges_a_repeat_split_by_blank():
    """'a' blank 'a' is the prefix (a, a), 'a' 'a' is (a,): the best prefix needs the merge rule and the blank path."""
    lp = torch.full((3, 3), -20.0)
    lp[0, 1] = lp[2, 1] = math.log(0.9)
    lp[1, 0] = math.log(0.9)
    lp = torch.log_softmax(lp, dim=-1).double()
    frames = [ctc_ref.frame_topk(lp[t].tolist(), 3) for t in range(3)]
    best, score = ctc_ref.prefix_beam_search(frames, beam=4)[0]
    assert best == (1, 1)
    assert abs(score - ctc_ref.prefix_marginals(lp.tolist())[(1, 1)]) < 1e-9


def test_prefix_beam_tie_break_is_candidate_order():
    """Equal scores: the earlier candidate (slot, then keep-before-extend, then top-K rank) wins."""
    lp = [[math.log(0.25)] * 4]
    frames = [ctc_ref.frame_topk(lp[0], 4)]
    assert [p for p, _ in ctc_ref.prefix_beam_search(frames, beam=3)] == [(), (1,), (2,)]


def _small_ctc_params(encoder_type='transformer'):
    c = torch.load(GOLDEN, weights_only=False)
    return copy.deepcopy(c['train'][encoder_type]['params'])


def test_registry_builds_the_reference_keys(fixture):
    from opentransformer_b200.model import CTCModel, End2EndModel
    assert End2EndModel['ctc'] is CTCModel
    base = fixture['baseline']
    m = End2EndModel['ctc'](base['params'])
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == base['shapes']
    for e in ('transformer', 'conformer'):
        c = fixture['train'][e]
        m = CTCModel(c['params'])
        assert {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in m.state_dict().items()} == c['sd_shapes']


def test_checkpoint_round_trip(tmp_path):
    from opentransformer_b200.model import CTCModel
    p = _small_ctc_params('conformer')
    torch.manual_seed(0)
    a = CTCModel(p)
    path = str(tmp_path / 'ctc.pt')
    a.save_checkpoint({'model': p}, path)
    chk = torch.load(path, weights_only=False)
    assert set(chk) == {'params', 'frontend', 'encoder', 'ctc'}
    torch.manual_seed(1)
    b = CTCModel(p)
    b.load_model(chk)
    sa, sb = a.state_dict(), b.state_dict()
    assert set(sa) == set(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)


def test_build_recognizer_returns_a_ctc_recognizer():
    from opentransformer_b200.model import CTCModel
    from opentransformer_b200.recognize import CTCRecognizer, build_recognizer
    args = SimpleNamespace(lm_weight=0.1, ngram_lm=None, beam_width=5, ngpu=0, mode='beam', alpha=0.1, beta=0.0)
    rec = build_recognizer('ctc', CTCModel(_small_ctc_params()), None, args, {i: str(i) for i in range(30)})
    assert isinstance(rec, CTCRecognizer) and rec.mode == 'beam' and rec.beam_width == 5 and not rec.model.training


def test_ngram_lm_is_refused():
    from opentransformer_b200.model import CTCModel
    from opentransformer_b200.recognize import CTCRecognizer
    with pytest.raises(NotImplementedError, match='KenLM'):
        CTCRecognizer(CTCModel(_small_ctc_params()), ngram_lm='lm.arpa', ngpu=0, mode='beam')


def test_lookahead_steps_is_refused():
    from opentransformer_b200.model import CTCModel
    p = _small_ctc_params()
    p['lookahead_steps'] = 2
    with pytest.raises(NotImplementedError, match='lookahead'):
        CTCModel(p)


def test_96_wide_heads_are_refused_in_training_before_device_work():
    """conformer_baseline.yaml's encoder (d_model 384, 4 heads) under a CTC head: the TrainPack message, raised by the
    shared encoder pack before any CUDA call (the tensors are on the CPU)."""
    from opentransformer_b200.model import CTCModel
    p = copy.deepcopy(CONFORMER_BASELINE)
    p = {'type': 'ctc', 'frontend_type': 'conv', 'encoder_type': 'conformer', 'frontend': p['frontend'], 'encoder': p['encoder'],
         'encoder_output_size': p['encoder']['d_model'], 'vocab_size': 40}
    m = CTCModel(p).train()
    x, mask = torch.zeros(1, 40, p['frontend']['input_size']), torch.ones(1, 40, dtype=torch.bool)
    tgt, tlen = torch.tensor([[1, 5, 6, 1]]), torch.tensor([3])
    with pytest.raises(NotImplementedError, match='training path: 64-wide attention heads only; the encoder has d_model 384 with 4 heads'):
        m({'inputs': x, 'mask': mask}, {'targets': tgt, 'targets_length': tlen})


def test_targets_length_is_required():
    from opentransformer_b200 import train
    from opentransformer_b200.model import CTCModel
    m = CTCModel(_small_ctc_params()).train()
    x, mask, tgt = torch.zeros(1, 40, 20), torch.ones(1, 40, dtype=torch.bool), torch.tensor([[1, 5, 6, 1]])
    with pytest.raises(ValueError, match='targets_length'):
        m({'inputs': x, 'mask': mask}, {'targets': tgt})
    tr = train.FusedTrainer(m, use_graph=False)
    with pytest.raises(TypeError, match='truth_length is required'):
        tr.step(x, mask, tgt)


def test_dropout_sites_of_a_ctc_model_are_the_encoders():
    from opentransformer_b200 import train
    from opentransformer_b200.model import CTCModel
    for e, n in (('transformer', 2), ('conformer', 3)):
        p = _small_ctc_params(e)
        p['encoder']['residual_dropout'] = 0.1
        sites = train.dropout_sites(CTCModel(p))
        assert [s for s, _, _ in sites] == list(range(train.ENC_SITE, train.ENC_SITE + 2 * n))
        assert all(part == 'encoder' and r == 0.1 for _, part, r in sites)


def test_decode_wrappers_check_shapes_before_any_device_work():
    """Mismatched operands raise in the ops wrappers instead of reading out of bounds (CPU tensors: no CUDA call is made)."""
    from opentransformer_b200 import ops
    B, T, K = 2, 5, 4
    n = torch.full((B,), T, dtype=torch.int32)
    lp, tok = torch.zeros(B * T, K), torch.zeros(B * T, K, dtype=torch.int32)
    with pytest.raises(ValueError, match='logits'):
        ops.ctc_frame_topk(torch.zeros(B * T - 1, 40), B, T, 40, n, K)
    with pytest.raises(ValueError, match='logits'):
        ops.ctc_frame_topk(torch.zeros(B * T, 32), B, T, 40, n, K)
    with pytest.raises(ValueError, match='in_len'):
        ops.ctc_frame_topk(torch.zeros(B * T, 40), B, T, 40, n[:1], K)
    with pytest.raises(ValueError, match='top_lp and top_id'):
        ops.ctc_greedy(lp[:, :1], tok, B, T, n)
    with pytest.raises(ValueError, match='top_lp and top_id'):
        ops.ctc_prefix_beam(lp[1:], tok[1:], B, T, n, 4)
    with pytest.raises(ValueError, match='in_len'):
        ops.ctc_prefix_beam(lp, tok, B, T, n[:1], 4)
