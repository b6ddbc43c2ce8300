"""Sampling-based MWER (DESIGN.md 4.11) restated in float64 -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Sampling.  Row n of a step draws token = argmax_v (x_v + g_v), v < V, ties to the lower id, with g_v = -log(-log u) and
    u(seed, step, n, v) = rng_u01(rng_key(rng_key(rng_key(seed, step), n), v))
in csrc/counter_rng.cuh's functions: mix32 is lowbias32, rng_key(s, c) = mix32(mix32(s) ^ c), and rng_u01(h) =
((h >> 9) + 0.5) * 2^-23, exact in fp32 and never 0 or 1.  They are restated here bit for bit in numpy uint32.  The row adds
x_token - logsumexp(x[:V]) to its score; drawing <S/E> (id 1) ends it, and an ended row emits <S/E>, keeps its score and
is its own parent, as every row is.

Estimator.  For utterance b with K samples y_k (cut at their first <S/E>) and edit distances W_k to the reference:
W^_b = mean_k W_k is the reported loss and c_k = (W_k - W^_b) / (K B) * grad_scale the coefficient of the sequence
log-probability l_k in the gradient, sum_b sum_k c_k dl_k: the score-function estimate of the gradient of E[W].
"""
import numpy as np
import torch

EOS = 1


def mix32(x):
    """lowbias32 on numpy uint32 (arrays or scalars); wrapping multiplication as the device's."""
    x = np.asarray(x, dtype=np.uint32)
    with np.errstate(over='ignore'):
        x = x ^ (x >> np.uint32(16))
        x = (x * np.uint32(0x7FEB352D)).astype(np.uint32)
        x = x ^ (x >> np.uint32(15))
        x = (x * np.uint32(0x846CA68B)).astype(np.uint32)
        x = x ^ (x >> np.uint32(16))
    return x


def rng_key(seed, counter):
    return mix32(mix32(np.asarray(seed, dtype=np.uint32)) ^ np.asarray(counter, dtype=np.uint32))


def rng_u01(h):
    """float64 of the fp32 uniform: (k + 0.5) / 2^23 with k the top 23 bits, exact in both precisions."""
    return ((np.asarray(h, dtype=np.uint32) >> np.uint32(9)).astype(np.float64) + 0.5) * 2.0 ** -23


def uniforms(seed, step, n, V):
    """u(seed, step, n, v) for v < V (float64 [V])."""
    s = np.uint32(np.int64(seed) & 0xFFFFFFFF)
    k = rng_key(rng_key(s, np.uint32(step)), np.uint32(n))
    return rng_u01(rng_key(k, np.arange(V, dtype=np.uint32)))


def gumbel(u):
    return -np.log(-np.log(u))


def draw(x, seed, step, n):
    """One row's draw in float64: x float [V] (may hold -inf) -> (token, x_token - logsumexp(x), the perturbed values).
    A row without a finite logit draws token 0 with increment -inf."""
    x = np.asarray(x, dtype=np.float64)
    V = x.shape[0]
    z = x + gumbel(uniforms(seed, step, n, V))
    if not np.isfinite(x).any():
        return 0, float('-inf'), z
    tok = int(np.argmax(z))                 # numpy's argmax takes the first (lowest) index of the maximum
    m = x[np.isfinite(x)].max()
    lse = m + np.log(np.exp(x[np.isfinite(x)] - m).sum())
    return tok, float(x[tok] - lse), z


def step(logits, V, flag, scores, seed, step_no):
    """One sampling step over all rows: logits float [N, >= V], flag bool [N], scores float64 [N] -> (tokens [N], new
    flag, new scores, perturbed values [N, V] of the live rows (None for ended rows))."""
    N = logits.shape[0]
    toks, zs = np.zeros(N, dtype=np.int64), []
    flag, scores = flag.copy(), scores.copy()
    for n in range(N):
        if flag[n]:
            toks[n] = EOS
            zs.append(None)
            continue
        t, inc, z = draw(logits[n, :V], seed, step_no, n)
        toks[n] = t
        scores[n] += inc
        flag[n] = t == EOS
        zs.append(z)
    return toks, flag, scores, zs


def sample_coefficients(W, B, grad_scale=1.0):
    """(W^ [B'], c [B', K]) of the errors W [B', K] (float64), c = (W - W^) / (K B) * grad_scale."""
    W = torch.as_tensor(W, dtype=torch.float64)
    K = W.shape[1]
    mean = W.mean(dim=1, keepdim=True)
    return mean.squeeze(1), (W - mean) / (K * B) * grad_scale
