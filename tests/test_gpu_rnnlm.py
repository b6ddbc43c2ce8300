"""The recurrent language model on the GPU (opentransformer_b200.lm.RecurrentLanguageModel, csrc/lstm.cu) against the fp32
restatement of the reference's recurrent LM (tests/rnnlm_ref.py, pinned to the reference by tests/test_rnnlm_ref.py).

Tolerances: the oracle's policy='bf16' rounds x, h and the weights where the CUDA path stores bf16, so what remains is fp32
summation order plus the odd bf16 rounding flip of h carried through the recurrence: 1e-2 relative L2 on log-probs and
states.  Gradients also round dG and the back-propagated activation gradients to bf16 (the oracle's autograd keeps them
fp32): 3e-2 relative L2 per parameter."""
import ctypes
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

if torch.cuda.is_available():
    from opentransformer_b200 import _lib, ops
    from opentransformer_b200.lm import RNNLM_SITE, RecurrentLanguageModel
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer, lm_log_probs
    DEV = torch.device('cuda:0')

from oracle import beam_search as obs
from oracle import speech_model as om
from tests import rnnlm_ref as rr
from tests.test_rnnlm_ref import FIXTURE, RNNLM_YAML, synth_state_dict

REL_STATES = 1e-2
REL_GRADS = 3e-2


def _rel(a, b):
    return float((a.float().cpu() - b.float()).norm() / b.float().norm())


def _lm(H, V=50, layers=2, tied=False, dropout=0.0, seed=0):
    torch.manual_seed(seed)
    params = dict(type='rnn_lm', vocab_size=V, num_layers=layers, hidden_size=H, residual_dropout=0.1, smoothing=0.1,
                  dropout=dropout, share_embedding=tied)
    lm = RecurrentLanguageModel(params)
    with torch.no_grad():
        lm.output_project.bias.normal_(0.0, 0.1)
    sd = {k: v.detach().clone().float() for k, v in lm.state_dict().items()}
    return lm.to(DEV), sd, params


def _tokens(N, L, V, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(2, V, (N, L), generator=g)


@pytest.mark.parametrize('L', [1, 7, 64])
@pytest.mark.parametrize('B', [1, 16, 37])
@pytest.mark.parametrize('H', [64, 1024])
def test_recurrence_forward(H, B, L):
    """predict() of a 2-layer LM: log-probs and (h_n, c_n) with the zero state and with a given (h0, c0)."""
    lm, sd, _ = _lm(H)
    lm.eval()
    tok = _tokens(B, L, 50, seed=H + B + L)
    g = torch.Generator().manual_seed(2)
    hidden = (0.5 * torch.randn(2, B, H, generator=g), 0.5 * torch.randn(2, B, H, generator=g))
    for hid in (None, hidden):
        ref_lp, (ref_h, ref_c) = rr.rnn_lm_predict(tok, sd, '', 2, hidden=hid, policy='bf16')
        lp, (h, c) = lm.predict(tok.to(DEV), None if hid is None else tuple(t.to(DEV) for t in hid))
        assert lp.shape == (B, L, 50) and h.shape == c.shape == (2, B, H) and h.dtype == torch.float32
        assert _rel(lp, ref_lp) < REL_STATES and _rel(h, ref_h) < REL_STATES and _rel(c, ref_c) < REL_STATES, (hid is None)


def test_carried_state_equals_one_call():
    """L one-token calls that carry (h, c) compute what one call over the L tokens does: the carried h_n is fp32 and is
    rounded to bf16 where the kernel stages it, exactly as h_t is inside one call; only the GEMM row count differs."""
    lm, _, _ = _lm(256, V=60)
    lm.eval()
    tok = _tokens(12, 9, 60).to(DEV)
    lp, (h, c) = lm.predict(tok)
    hid, steps = None, []
    for t in range(tok.shape[1]):
        lpt, hid = lm.predict(tok[:, t:t + 1], hid)
        steps.append(lpt)
    assert torch.allclose(torch.cat(steps, 1), lp, rtol=0, atol=1e-4)
    assert torch.allclose(hid[0], h, rtol=0, atol=1e-5) and torch.allclose(hid[1], c, rtol=0, atol=1e-5)


def _batch(N, L, V, seed=3):
    tok = _tokens(N, L + 1, V, seed)
    inputs, targets = tok[:, :-1].clone(), tok[:, 1:].clone()
    for b in range(1, N):                      # PAD-padded tails of different lengths
        n = max(1, L - 3 * b)
        inputs[b, n:] = 0
        targets[b, n:] = 0
    return inputs, targets


def _train_grads(lm, inputs, targets):
    lm.train()
    lm.zero_grad(set_to_none=True)
    loss, none = lm({'inputs': inputs.to(DEV)}, {'targets': targets.to(DEV)})
    assert none is None
    loss.backward()
    return loss.detach(), {n: p.grad for n, p in lm.named_parameters()}


def _check_grads(loss, grads, ref_loss, ref_grads):
    assert abs(float(loss) - float(ref_loss)) < 1e-3 * abs(float(ref_loss)) + 1e-4
    assert set(grads) == set(ref_grads)
    for k, ref in ref_grads.items():
        assert grads[k] is not None and torch.isfinite(grads[k]).all(), k
        r = _rel(grads[k], ref)
        assert r < REL_GRADS, f'{k}: rel_l2 {r:.3e}'


@pytest.mark.parametrize('H,V,tied', [(64, 40, False), (64, 40, True), (1024, 4233, True)])
def test_backward_against_oracle(H, V, tied):
    """The loss and every parameter gradient after loss.backward(), tied and untied, including the shipped H = 1024."""
    lm, sd, params = _lm(H, V=V, tied=tied)
    inputs, targets = _batch(5, 12, V)
    loss, grads = _train_grads(lm, inputs, targets)
    ref_loss, ref_grads = rr.rnn_lm_loss_and_grads(inputs, targets, {k: v for k, v in sd.items()}, params, policy='bf16')
    _check_grads(loss, grads, ref_loss, ref_grads)


def test_backward_with_dropout_replayed():
    """dropout 0.1 between the layers: the oracle replays the mask of the CUDA call (counter hash of (seed, site, row,
    col), time-major rows); two calls draw different masks."""
    lm, sd, params = _lm(64, V=40, layers=3, dropout=0.1)
    inputs, targets = _batch(6, 10, 40)
    N, L = inputs.shape
    masks = []
    for _ in range(2):
        loss, grads = _train_grads(lm, inputs, targets)
        seed = lm._drop_seed.clone()
        mk = {k: ops.dropout_mask(L * N, 64, 0.1, seed, RNNLM_SITE + k).cpu().float().view(L, N, 64).transpose(0, 1)
              for k in range(2)}
        masks.append(mk)
        om.set_dropout(lambda site, t, mk=mk: t * mk[site[1]] / 0.9)
        try:
            ref_loss, ref_grads = rr.rnn_lm_loss_and_grads(inputs, targets, sd, params, policy='bf16')
        finally:
            om.set_dropout(None)
        _check_grads(loss, grads, ref_loss, ref_grads)
    for k in range(2):
        assert not torch.equal(masks[0][k], masks[1][k])
        assert 0.85 < float(masks[0][k].mean()) < 0.95


def test_public_training_seam():
    lm, _, _ = _lm(128, V=70, tied=True, dropout=0.1)
    inputs, targets = _batch(4, 8, 70)
    loss, grads = _train_grads(lm, inputs, targets)
    assert torch.isfinite(loss)
    for n, p in lm.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape and torch.isfinite(p.grad).all(), n


def test_shipped_rnnlm_yaml_model():
    """rnnlm.yaml: load a state dict with the reference's key names, predict against the oracle, one training step."""
    keys = torch.load(FIXTURE)['rnnlm_yaml_keys']
    sd = {k: 0.1 * v for k, v in synth_state_dict(keys, 11, tied=True).items()}
    sd['output_project.weight'] = sd['embedding.weight']
    lm = RecurrentLanguageModel(RNNLM_YAML)
    lm.load_state_dict(sd, strict=True)
    lm = lm.to(DEV).eval()
    tok = _tokens(8, 20, 4233)
    ref_lp, (ref_h, ref_c) = rr.rnn_lm_predict(tok, sd, '', 2, policy='bf16')
    lp, (h, c) = lm.predict(tok.to(DEV))
    assert _rel(lp, ref_lp) < REL_STATES and _rel(h, ref_h) < REL_STATES and _rel(c, ref_c) < REL_STATES
    opt = torch.optim.Adam(lm.parameters(), lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6)
    inputs, targets = _batch(8, 20, 4233)
    lm.train()
    loss, _ = lm({'inputs': inputs.to(DEV)}, {'targets': targets.to(DEV)})
    loss.backward()
    torch.nn.utils.clip_grad_norm_(lm.parameters(), 5.0)
    opt.step()
    lm.eval()
    lp2, _ = lm.predict(tok.to(DEV))          # the bf16 pack follows the updated parameters
    assert torch.isfinite(loss) and torch.isfinite(lp2).all() and not torch.equal(lp, lp2)


def test_rnn_lm_shallow_fusion_lockstep():
    """Beam search with an RNN LM: every step the LM reads the newest token with no carried state (the reference passes
    cache['lm'] = None), and the oracle's beam_step fed the CUDA decoder's and the CUDA LM's log-probs makes the same
    integer decisions."""
    from tests.test_gpu_model import _batch as speech_batch, _build, _params
    lm, _, _ = _lm(256, V=4234, tied=True, seed=77)
    lm.eval()
    params = _params(n_enc=1, n_dec=2)
    model, _ = _build(params)
    B, beam, max_len, lmw = 2, 3, 6, 0.3
    x, mask = speech_batch(B, 160, 80, [160, 131])
    with torch.no_grad():
        mem, lens, _, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        bd = BeamDecoder(model.decoder, B, beam, T2, max_len, DEV, use_graph=False)
        bd.setup(mem, lens)
        bd.lm_weight = lmw
        preds = torch.full((B * beam, 1), 1, dtype=torch.long)
        scores = torch.tensor([0.0] + [float('-inf')] * (beam - 1)).repeat(B).unsqueeze(1)
        flag = torch.zeros_like(scores, dtype=torch.bool)
        for s in range(max_len):
            prefix = bd.state.reconstruct(s)
            bd.lm_logp = lm_log_probs(lm, prefix)
            assert torch.equal(bd.lm_logp, lm.predict(prefix[:, -1:])[0].squeeze(1))
            lm_cpu = bd.lm_logp.cpu()
            bd._step_kernels()
            dec_lp = bd.logp.cpu() - lmw * lm_cpu
            preds, scores, flag = obs.beam_step(dec_lp, preds, scores, flag, beam, lm_log_probs=lm_cpu, lm_weight=lmw)
            assert torch.equal(bd.state.reconstruct(s + 1).cpu(), preds), f'fusion: ids differ at step {s}'
    rec = SpeechToTextRecognizer(model, lm=lm, lm_weight=lmw, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1)
    ids, sc, n = rec.recognize_ids(x.to(DEV), mask.to(DEV))
    assert ids.shape == (B, 1, n)
    lp, hid = rec.lm_decode(torch.ones(B * beam, 3, dtype=torch.long, device=DEV))
    assert lp.shape == (B * beam, 1, 4234) and hid[0].shape == (2, B * beam, 256)


def test_refused_configurations_launch_nothing():
    """A hidden size the kernels do not take returns the error before any launch: the outputs keep their sentinel."""
    for H, msg in ((1020, b'multiple of 8'), (2048, b'does not fit')):
        L, B = 2, 3
        gx = torch.zeros(L * B, 4 * H, device=DEV)
        w = torch.zeros(4 * H, H, dtype=ops.BF16, device=DEV)
        y = torch.full((L * B, H), 7.0, dtype=ops.BF16, device=DEV)
        hn = torch.full((B, H), 7.0, device=DEV)
        cn = torch.full((B, H), 7.0, device=DEV)
        bar = torch.zeros(2, dtype=torch.int32, device=DEV)
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        rc = _lib.lib().otb_lstm_fwd(p(gx), p(w), None, None, p(y), p(hn), p(cn), None, None, p(bar), L, B, H, st)
        assert rc == 1 and msg in _lib.lib().otb_last_error()
        torch.cuda.synchronize()
        assert bool((y == 7).all()) and bool((hn == 7).all()) and bool((cn == 7).all()) and bool((bar == 0).all())
    with pytest.raises(NotImplementedError, match='does not fit'):
        _lm(2048, V=16)[0].predict(torch.ones(1, 1, dtype=torch.long, device=DEV))
