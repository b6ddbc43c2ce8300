"""LM shallow fusion in the transducer's greedy and ALSD searches (DESIGN.md 4.22) restated in float64 -- TEST
INFRASTRUCTURE, NOT PRODUCT CODE.

lp(b, t, y) -> float64 [V] is the joint's log-probs at frame t after labels y (rnnt_beam_ref's callback); lm(b, y) ->
float64 [V] is log p_lm(. | <S/E>, y).  A label k taken after labels y scores lp(k) + (lm_weight * lm(y)[k] + beta); blank
scores lp(blank) alone.  At lm_weight 0 the LM row is not read.  fused_row() folds that into one row, so the unfused
ALSD restatement (rnnt_beam_ref.step), which ranks labels by their row value and scores blank by column 0, runs the fused
search unchanged.  Only the early end differs: with beta > 0 a live hypothesis with u labels may still gain
beta (max_len - u), and the bound is logsumexp(s + beta (max_len - u)).
"""
import math

import numpy as np

from tests import rnnt_beam_ref as beam_ref


def fused_row(lp_row, lm_row, lm_weight, beta):
    """float64 [V]: column 0 (blank) lp_row[0], label k lp_row[k] + (lm_weight * lm_row[k] + beta)."""
    term = np.full(len(lp_row), float(beta)) if lm_weight == 0 else lm_weight * np.asarray(lm_row, np.float64) + beta
    out = np.asarray(lp_row, np.float64) + term
    out[0] = lp_row[0]
    return out


def end_bound(utt, beta, max_len):
    """logsumexp over live slots of s + beta (max_len - u) (beta > 0), or of s alone."""
    live = [s[0] + (beta * (max_len - s[1]) if beta > 0 else 0.0) for s in utt.slots if s is not None]
    m = max(live)
    return m + math.log(sum(math.exp(v - m) for v in live))


def alsd_step(utt, lp, lm, W, max_len, lm_weight, beta, early=True):
    """One fused step of utt; lp[j] / lm[j] the joint's and the LM's rows of live slot j -> (par, tok) as
    rnnt_beam_ref.step."""
    rows = {j: fused_row(lp[j], lm[j], lm_weight, beta) for j in lp}
    par, tok = beam_ref.step(utt, rows, W, max_len, early=False)
    if early and not utt.done and len(utt.finals) == W and any(s is not None for s in utt.slots):
        utt.done = end_bound(utt, beta, max_len) <= utt.finals[-1][0]
    return par, tok


def alsd_search(lp_fn, lm_fn, t_len, K, W, max_len, lm_weight, beta, early=True):
    """The whole fused ALSD search of each utterance b -> [rnnt_beam_ref.Utterance] (ended)."""
    out = []
    for b, T in enumerate(t_len):
        utt = beam_ref.Utterance(K, int(T))
        while not utt.done:
            live = {j: s for j, s in enumerate(utt.slots) if s is not None}
            lp = {j: lp_fn(b, s[2], utt.labels(s[3])) for j, s in live.items()}
            lm = {j: lm_fn(b, utt.labels(s[3])) for j, s in live.items()}
            alsd_step(utt, lp, lm, W, max_len, lm_weight, beta, early)
        out.append(utt)
    return out


def greedy_step(state, lp_row, lm_row, T, max_len, max_sym, lm_weight, beta):
    """One fused greedy step of one utterance.  state: dict(frame, n_sym, y (list), score, done).  The arg-max of the fused
    row (ties to the lower id); blank when the row may not emit.  A label adds its fused value, blank its log-prob."""
    if state['done']:
        return
    row = fused_row(lp_row, lm_row, lm_weight, beta)
    k = int(np.argmax(row))
    if state['n_sym'] >= max_sym or len(state['y']) >= max_len:
        k = 0
    state['score'] += row[k]
    if k:
        state['y'].append(k)
        state['n_sym'] += 1
    else:
        state['frame'] += 1
        state['n_sym'] = 0
        state['done'] = state['frame'] >= T


def greedy_search(lp_fn, lm_fn, t_len, max_len, max_sym, lm_weight, beta):
    """-> [(labels tuple, fused score)] per utterance."""
    out = []
    for b, T in enumerate(t_len):
        st = dict(frame=0, n_sym=0, y=[], score=0.0, done=T <= 0)
        while not st['done']:
            y = tuple(st['y'])
            greedy_step(st, lp_fn(b, st['frame'], y), lm_fn(b, y), T, max_len, max_sym, lm_weight, beta)
        out.append((tuple(st['y']), st['score']))
    return out


def synthetic_lm(seed, V, scale=1.5, context_free=False):
    """A callback log p_lm(. | <S/E>, y): a log-softmax of normal logits drawn from (seed, b, y), or from (seed, b) alone
    when context_free."""
    cache = {}

    def lm(b, y):
        key = (b,) if context_free else (b, tuple(y))
        if key not in cache:
            g = np.random.default_rng([seed, 7, b] + ([] if context_free else [len(y)] + list(y)))
            x = scale * g.standard_normal(V)
            m = x.max()
            cache[key] = x - (m + math.log(np.exp(x - m).sum()))
        return cache[key]
    return lm
