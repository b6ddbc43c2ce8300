"""CPU checks of the sampling restatement (tests/mwer_sample_ref.py) that the GPU tests compare otb_sample_step,
sample_ids and the sampled MWER pass with: the numpy hash against csrc/counter_rng.cuh compiled for the host, the Gumbel-max
draw against softmax, the sampled coefficients against autograd and against the exact gradient of the expected risk, and
the refusals of the sampling decoder, sample_ids, forward_backward and FusedTrainer before any device work."""
import itertools
import os
import subprocess
import types

import numpy as np
import pytest
import torch

from tests import mwer_sample_ref as sr
from tests.test_ctc_model_ref import _small_ctc_params
from tests.test_mwer_ref import _speech_params
from tests.test_transformer_lm_ref import _cuda_calls_fail

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (seed, counter) -> (rng_key, rng_u01) printed by the header's functions compiled for the host
PINNED = [(0, 5, 1548080446, 0.360440552), (1, 982, 792904711, 0.184612572), (123456789, 1959, 3329044626, 0.775103629),
          (4294967295, 5, 2683073441, 0.624701679)]

_HOST_PROBE = r'''
#include <stdio.h>
#include "counter_rng.cuh"
int main() {
    unsigned s, c;
    while (scanf("%u %u", &s, &c) == 2) {
        const unsigned h = otb::rng_key(s, c);
        printf("%u %a\n", h, (double)otb::rng_u01(h));
    }
    return 0;
}
'''


def test_hash_matches_pinned_values():
    for s, c, h, u in PINNED:
        assert int(sr.rng_key(s, c)) == h
        assert abs(float(sr.rng_u01(h)) - u) < 1e-9


def test_hash_matches_the_header_compiled_for_the_host(tmp_path):
    from opentransformer_b200 import build
    src = tmp_path / 'probe.cu'
    src.write_text(_HOST_PROBE)
    exe = tmp_path / 'probe'
    subprocess.run([build._nvcc(), '-I', os.path.join(ROOT, 'opentransformer_b200', 'csrc'), str(src), '-o', str(exe)],
                   check=True, capture_output=True)
    rng = np.random.default_rng(0)
    seeds = np.concatenate([[0, 1, 0xFFFFFFFF, 0x80000000], rng.integers(0, 2 ** 32, 300)]).astype(np.uint32)
    counters = np.concatenate([[0, 1, 0xFFFFFFFF, 49151], rng.integers(0, 2 ** 32, 300)]).astype(np.uint32)
    out = subprocess.run([str(exe)], input=''.join(f'{s} {c}\n' for s, c in zip(seeds, counters)), text=True,
                         capture_output=True, check=True).stdout.split('\n')
    for (s, c), line in zip(zip(seeds, counters), out):
        h, u = line.split()
        assert int(sr.rng_key(s, c)) == int(h), (s, c)
        assert float(sr.rng_u01(int(h))) == float.fromhex(u), (s, c)
    # the sampling layout: u(seed, step, n, v) chains three keys
    k = sr.rng_key(sr.rng_key(np.uint32(7), np.uint32(3)), np.uint32(2))
    assert np.array_equal(sr.uniforms(7, 3, 2, 5), sr.rng_u01(sr.rng_key(k, np.arange(5, dtype=np.uint32))))
    u = sr.uniforms(-1, 0, 0, 4096)               # a negative int32 seed is its 32 bits
    assert np.array_equal(u, sr.uniforms(0xFFFFFFFF, 0, 0, 4096)) and 0.0 < u.min() and u.max() < 1.0


@pytest.mark.parametrize('x', [[0.0, 0.0, 0.0], [2.0, 0.5, -1.0, 0.0], [1.0, float('-inf'), 0.3, -0.7, 2.2, 0.0]])
def test_gumbel_max_draw_follows_softmax(x):
    """20000 draws over (step, row) counters at a fixed seed: the Pearson chi-square of the token counts against
    softmax(x) stays under the 0.999 quantile of its distribution (so the test is deterministic and not fragile)."""
    from scipy.stats import chi2
    x = np.asarray(x)
    V, steps, rows = x.shape[0], 200, 100
    counts = np.zeros(V)
    for s in range(steps):
        for n in range(rows):
            counts[sr.draw(x, 2024, s, n)[0]] += 1
    p = np.exp(x - x.max())
    p /= p.sum()
    live = p > 0
    assert counts[~live].sum() == 0, 'a -inf logit was drawn'
    e = p[live] * steps * rows
    stat = float(((counts[live] - e) ** 2 / e).sum())
    assert stat < chi2.ppf(0.999, live.sum() - 1), (stat, counts, e)


def test_draw_is_the_perturbed_argmax_and_the_increment_the_log_prob():
    x = np.full(6, float('-inf'))
    x[[4, 1]] = 2.0 ** 30                 # x + g rounds to 2^30 in fp32 but not in float64: no tie in this restatement
    tok, inc, z = sr.draw(x, 3, 0, 0)
    assert tok == (1 if z[1] >= z[4] else 4) and abs(inc + np.log(2.0)) < 1e-6
    x = np.array([0.3, -1.2, 2.0])
    tok, inc, z = sr.draw(x, 11, 5, 7)
    assert tok == int(np.argmax(z)) and abs(inc - (x[tok] - np.log(np.exp(x).sum()))) < 1e-12
    assert sr.draw(np.full(3, float('-inf')), 0, 0, 0)[:2] == (0, float('-inf'))


def test_step_keeps_ended_rows_and_their_scores():
    logits = np.random.default_rng(1).normal(size=(4, 7))
    flag = np.array([False, True, False, True])
    scores = np.array([0.0, -3.0, -1.0, -2.5])
    toks, f2, s2, zs = sr.step(logits, 7, flag, scores, 5, 2)
    assert toks[1] == sr.EOS and toks[3] == sr.EOS and s2[1] == -3.0 and s2[3] == -2.5 and f2[1] and f2[3]
    for n in (0, 2):
        t, inc, _ = sr.draw(logits[n], 5, 2, n)
        assert toks[n] == t and s2[n] == scores[n] + inc and f2[n] == (t == sr.EOS)


@pytest.mark.parametrize('seed', range(3))
def test_sampled_coefficients_through_autograd_equal_the_closed_form(seed):
    """S = sum_k c_k l_k with c detached: its logits gradient is c_k (onehot(y'_t) - softmax(x_t)) row by row, the form
    otb_mwer_grad writes."""
    g = torch.Generator().manual_seed(seed)
    B, K, Lp, V = 2, 4, 5, 9
    logits = torch.randn(B, K, Lp, V, generator=g, dtype=torch.float64, requires_grad=True)
    n = torch.randint(0, Lp, (B, K), generator=g)
    tgt = torch.randint(0, V, (B, K, Lp), generator=g)
    W = torch.randint(0, 5, (B, K), generator=g).double()
    W[1] = 3.0                                              # an utterance with all W equal: exactly zero
    mean, c = sr.sample_coefficients(W, B, grad_scale=0.5)
    assert torch.equal(mean, W.mean(dim=1)) and torch.equal(c[1], torch.zeros(K, dtype=torch.float64))
    lp = torch.log_softmax(logits, dim=-1).gather(-1, tgt[..., None]).squeeze(-1)
    live = torch.arange(Lp) <= n[..., None]
    l = (lp * live).sum(dim=2)
    (c.detach() * l).sum().backward()
    closed = c[..., None, None] * (torch.nn.functional.one_hot(tgt, V) - torch.softmax(logits.detach(), dim=-1))
    closed = closed * live[..., None]
    torch.testing.assert_close(logits.grad, closed, rtol=1e-12, atol=1e-14)


def test_sampled_estimator_expectation_by_enumeration():
    """On a one-step model, p = softmax(theta) over 3 tokens with error W(y): the expectation of the K-sample estimate
    sum_k (W_k - mean W) / K * dlog p(y_k) over all K-tuples equals (1 - 1/K) * d E[W] / d theta.  The mean includes the
    sample itself, which scales the estimate by (K - 1) / K and leaves its direction unbiased."""
    theta = torch.tensor([0.4, -0.3, 1.1], dtype=torch.float64, requires_grad=True)
    Wtok = torch.tensor([2.0, 0.0, 5.0], dtype=torch.float64)
    p = torch.softmax(theta, 0)
    (exact,) = torch.autograd.grad((p * Wtok).sum(), theta)
    pd = p.detach()
    for K in (2, 3):
        est = torch.zeros(3, dtype=torch.float64)
        for ys in itertools.product(range(3), repeat=K):
            prob = torch.prod(pd[list(ys)])
            W = Wtok[list(ys)][None]
            _, c = sr.sample_coefficients(W, 1)
            for k, y in enumerate(ys):
                est += prob * c[0, k] * (torch.nn.functional.one_hot(torch.tensor(y), 3) - pd)
        torch.testing.assert_close(est, (1 - 1 / K) * exact, rtol=1e-12, atol=1e-14)


class _FakeLM(types.SimpleNamespace):
    def eval(self):
        return self


def test_sampling_refusals_come_before_device_work(monkeypatch):
    from opentransformer_b200 import train
    from opentransformer_b200.model import CTCModel, SpeechToText
    from opentransformer_b200.recognize import BeamDecoder, SpeechToTextRecognizer
    speech, joint, ctc_model = SpeechToText(_speech_params()), SpeechToText(_speech_params(0.3)), CTCModel(_small_ctc_params())
    lm = _FakeLM(model_type='transformer_lm', vocab_size=40)
    x, mask = torch.zeros(1, 8, 80), torch.ones(1, 8, dtype=torch.bool)
    _cuda_calls_fail(monkeypatch)
    # the decoder
    for kw in ({'lm': (lm, 0.3)}, {'ctc': (None, 0.3, 4)}):
        with pytest.raises(NotImplementedError, match='sampling'):
            BeamDecoder(speech.decoder, 1, 2, 8, 5, torch.device('cpu'), sample=True, **kw)
    # the public call
    for rec in (SpeechToTextRecognizer(speech, lm=lm, ngpu=0), SpeechToTextRecognizer(joint, ctc_weight=0.3, ngpu=0),
                SpeechToTextRecognizer(joint, apply_rescoring=True, ngpu=0)):
        with pytest.raises(NotImplementedError, match='sample_ids'):
            rec.sample_ids(x, mask, 4, 0)
    rec = SpeechToTextRecognizer(speech, ngpu=0)
    for k in (0, 17, -1, 2.0):
        with pytest.raises(ValueError, match='num_samples'):
            rec.sample_ids(x, mask, k, 0)
    # training
    with pytest.raises(ValueError, match='mwer_estimator'):
        train.forward_backward(speech, x, mask, torch.ones(1, 3, dtype=torch.long), mwer_estimator='beam')
    with pytest.raises(NotImplementedError, match='attention decoder'):
        train.FusedTrainer(ctc_model, mwer_samples=4)
    for k in (1, 17, -2):
        with pytest.raises(ValueError, match='mwer_samples'):
            train.FusedTrainer(speech, mwer_samples=k)
    with pytest.raises(ValueError, match='choose one'):
        train.FusedTrainer(speech, mwer_samples=4, mwer_nbest=4)
    with pytest.raises(NotImplementedError, match='MixSpeech'):
        train.FusedTrainer(speech, mwer_samples=4, mixspeech=True)
