"""The transducer's ALSD beam search (DESIGN.md 4.22) restated in float64 -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Utterance keeps the state the kernel keeps: K slots (score, u, frame, node) or None, the node table [(parent, token)]
with node 0 the empty sequence, and the n-best F [(score, step, slot, node, u)].  step() is one search step of one
utterance over the log-probs lp[j] (float64 [V]) of each live slot j; search() runs whole utterances over a callback
lp(b, t, y) -> float64 [V], the log-probs of the joint at frame t after the labels y (a tuple).

The rules: a live hypothesis at frame t < T forms a blank candidate (a final when t + 1 = T) and, while u < max_len, one
candidate for each of its min(K, V - 1) best labels (ties to the lower id).  A label candidate with the labels of a live
blank candidate is log-added into it and takes its place.  The K best candidates (score descending, ties in formation
order: parent slot, blank before labels, labels in top-k order) are the next slots.  F keeps the W best finals (ties to the
earlier step, then the lower slot).  The utterance ends when no slot is live, or (early) F is full and the logsumexp of the
live scores is no more than F's worst.
"""
import math

import numpy as np

NEG = float('-inf')


def _logaddexp(a, b):
    m = max(a, b)
    return m + math.log1p(math.exp(-abs(a - b)))


class Utterance:
    def __init__(self, K, T):
        self.K, self.T = K, T
        self.slots = [None] * K
        if T >= 1:
            self.slots[0] = (0.0, 0, 0, 0)
        self.nodes = [(-1, 0)]
        self.finals = []
        self.done = False
        self.steps = 0
        # what the sweep counts: merges, merges of a prefix that sits on another node than the label's parent (found only
        # by comparing strings), and nodes made for a string that already had one (a prefix formed again)
        self.merges = self.string_merges = self.recreated = 0
        self._strings = {()}

    def labels(self, node):
        out = []
        while node != 0:
            node, tok = self.nodes[node]
            out.append(tok)
        return tuple(reversed(out))

    def nbest(self, W):
        """-> [(labels, score)] best first, W entries: (() , -inf) past the finals found."""
        out = [(self.labels(f[3]), f[0]) for f in self.finals]
        return out + [((), NEG)] * (W - len(out))


def top_labels(lp, K):
    """The min(K, V - 1) best labels of lp (float64 [V]), ties to the lower id."""
    V = len(lp)
    return sorted(range(1, V), key=lambda k: (-lp[k], k))[:min(K, V - 1)]


def step(utt, lp, W, max_len, early=True):
    """One search step of utt; lp[j] the log-probs of live slot j.  -> (par, tok) per new slot: its parent slot and the
    label it took (0: blank or empty; an empty slot's parent is itself)."""
    K, T = utt.K, utt.T
    if utt.done:
        return list(range(K)), [0] * K
    cands, new_finals = [], []
    for j, s in enumerate(utt.slots):
        if s is None:
            continue
        score, u, frame, node = s
        blank = score + float(lp[j][0])
        if frame + 1 == T:
            new_finals.append((blank, utt.steps, j, node, u))
        else:
            cands.append(dict(score=blank, j=j, tok=0, u=u, frame=frame + 1, node=node))
        if u < max_len:
            for k in top_labels(lp[j], K):
                cands.append(dict(score=score + float(lp[j][k]), j=j, tok=k, u=u + 1, frame=frame, node=None))
    # merge: the label candidates are y_j + [k], the blank candidates y_a
    blanks = {(utt.labels(c['node']), c['frame']): c for c in cands if c['tok'] == 0}
    kept = []
    for c in cands:
        if c['tok']:
            parent = utt.slots[c['j']][3]
            a = blanks.get((utt.labels(parent) + (c['tok'],), c['frame']))
            if a is not None:
                a['score'] = _logaddexp(a['score'], c['score'])
                utt.merges += 1
                utt.string_merges += utt.nodes[a['node']][0] != parent
                continue
        kept.append(c)
    order = sorted(range(len(kept)), key=lambda i: (-kept[i]['score'], i))[:K]
    sel = [kept[i] for i in order]
    utt.finals = sorted(utt.finals + new_finals, key=lambda f: (-f[0], f[1], f[2]))[:W]
    par, tok, slots = [], [], []
    for r in range(K):
        if r < len(sel):
            c = sel[r]
            node = c['node']
            if c['tok']:
                parent = utt.slots[c['j']][3]
                s = utt.labels(parent) + (c['tok'],)
                utt.recreated += s in utt._strings
                utt._strings.add(s)
                utt.nodes.append((parent, c['tok']))
                node = len(utt.nodes) - 1
            slots.append((c['score'], c['u'], c['frame'], node))
            par.append(c['j'])
            tok.append(c['tok'])
        else:
            slots.append(None)
            par.append(r)
            tok.append(0)
    utt.slots = slots
    utt.steps += 1
    live = [c['score'] for c in sel]
    if not live:
        utt.done = True
    elif early and len(utt.finals) == W:
        m = max(live)
        utt.done = m + math.log(sum(math.exp(v - m) for v in live)) <= utt.finals[-1][0]
    return par, tok


def search(lp_fn, t_len, K, W, max_len, early=True):
    """The whole search of each utterance b (t_len[b] frames) -> [Utterance] (ended)."""
    out = []
    for b, T in enumerate(t_len):
        utt = Utterance(K, int(T))
        while not utt.done:
            lp = {j: lp_fn(b, s[2], utt.labels(s[3])) for j, s in enumerate(utt.slots) if s is not None}
            step(utt, lp, W, max_len, early)
        out.append(utt)
    return out


def synthetic_lp(seed, V, scale=2.0, blank_bias=0.0):
    """A callback whose log-probs are a log-softmax of normal logits drawn from (seed, b, t, y): a lattice with no
    structure, where equal (b, t, y) always give the same row."""
    cache = {}

    def lp(b, t, y):
        key = (b, t, tuple(y))
        if key not in cache:
            g = np.random.default_rng([seed, b, t, len(y)] + list(y))
            x = scale * g.standard_normal(V)
            x[0] += blank_bias
            m = x.max()
            cache[key] = x - (m + math.log(np.exp(x - m).sum()))
        return cache[key]
    return lp
