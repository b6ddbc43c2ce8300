"""CTC prefix scoring and the joint CTC/attention beam step on the CPU, float64 -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A plain restatement of DESIGN.md 4.9 (csrc/ctc_prefix.cu is the product):

  - empty_prefix / extend: gamma and psi of a hypothesis, and of the hypothesis extended by each of a list of candidates;
  - prefix_state: the same for a whole token list, one token at a time;
  - enumerate_labels: every frame-level path of a tiny problem, collapsed, with its probability;
  - JointSearch: the beam search with the CTC term, one step at a time.  A step builds the [N, V] joint score matrix (-inf
    outside each row's P candidates) and hands it to the unchanged oracle.beam_search.beam_step; it also reports the
    smallest margin by which any of the step's decisions was taken.
"""
import itertools

import torch

from oracle.beam_search import beam_step

NEG_INF = float('-inf')
BLANK, EOS = 0, 1
F64 = torch.float64


def empty_prefix(lp, n_frames, blank=BLANK):
    """lp [T, V] of one utterance -> (gamma f64 [n_frames, 2] = {-inf, running sum of the blank column}, psi = 0)."""
    g = torch.full((n_frames, 2), NEG_INF, dtype=F64)
    g[:, 1] = lp[:n_frames, blank].double().cumsum(0)
    return g, torch.zeros((), dtype=F64)


def extend(lp, n_frames, gamma, empty, last, cands, blank=BLANK, eos=EOS):
    """gamma f64 [n_frames, 2] of a hypothesis g (`empty`: g has no token yet; `last`: its last token otherwise) ->
    (gamma f64 [P, n_frames, 2], psi f64 [P]) of g extended by each token of `cands`.  A candidate equal to `eos`
    completes the hypothesis: its psi is the log-probability of the whole label sequence; eos=None scores every
    candidate as a prefix.  The blank is not a label: extending by it gives -inf throughout."""
    c = torch.as_tensor(cands, dtype=torch.int64).view(-1)
    P = c.numel()
    x = lp[:n_frames].double()[:, c].clone()
    x[:, c == blank] = NEG_INF
    lb = lp[:n_frames, blank].double()
    same = (c == int(last)) if not empty else torch.zeros(P, dtype=torch.bool)
    out = torch.full((P, n_frames, 2), NEG_INF, dtype=F64)
    gn = torch.full((P,), NEG_INF, dtype=F64)
    gb = torch.full((P,), NEG_INF, dtype=F64)
    ph = torch.full((P,), 0.0 if empty else NEG_INF, dtype=F64)          # phi(-1)
    terms = []
    for t in range(n_frames):
        terms.append(ph + x[t])
        new_gn = torch.logaddexp(gn, ph) + x[t]
        gb = torch.logaddexp(gn, gb) + lb[t]
        gn = new_gn
        out[:, t, 0], out[:, t, 1] = gn, gb
        ph = torch.where(same, gamma[t, 1].expand(P), torch.logaddexp(gamma[t, 0], gamma[t, 1]).expand(P))
    psi = torch.logsumexp(torch.stack(terms), dim=0) if terms else torch.full((P,), NEG_INF, dtype=F64)
    if eos is not None:
        psi = torch.where(c == eos, torch.logaddexp(gn, gb), psi)
    return out, psi


def prefix_state(lp, n_frames, tokens, eos=EOS):
    """(gamma, psi) of the hypothesis `tokens`, built one token at a time."""
    gamma, psi = empty_prefix(lp, n_frames)
    for i, tok in enumerate(tokens):
        g, p = extend(lp, n_frames, gamma, i == 0, tokens[i - 1] if i else -1, [tok], eos=eos)
        gamma, psi = g[0], p[0]
    return gamma, psi


def total(gamma):
    """log P(labels == g) from gamma(g): both endings at the last frame."""
    return torch.logaddexp(gamma[-1, 0], gamma[-1, 1]) if gamma.shape[0] else torch.tensor(NEG_INF, dtype=F64)


def enumerate_labels(lp, blank=BLANK):
    """Every path of lp [T, V] (V ** T of them): {collapsed label tuple: probability}."""
    T, V = lp.shape
    p = lp.double().exp()
    out = {}
    for path in itertools.product(range(V), repeat=T):
        prob = 1.0
        for t, v in enumerate(path):
            prob *= float(p[t, v])
        labels = tuple(v for i, v in enumerate(path) if v != blank and (i == 0 or v != path[i - 1]))
        out[labels] = out.get(labels, 0.0) + prob
    return out


def _gap(sorted_desc):
    """Smallest difference between neighbours of a descending list; pairs of -inf do not count."""
    d = sorted_desc[:-1] - sorted_desc[1:]
    d = d[~torch.isnan(d)]
    return float(d.min()) if d.numel() else float('inf')


class JointSearch:
    """Beam search with the CTC prefix term (DESIGN.md 4.9) over lp f64 [B, T, V] with n_frames[b] valid frames.
    step(att_logp [N, V], lm_logp or None) advances preds / scores / flag as beam_step does and returns the smallest margin
    of the step's decisions among rows that can still win (finite score, not finished): the P-th against the (P+1)-th
    token of the pre-pruning, the beam-th against the (beam+1)-th candidate by the joint score, and neighbours among the
    utterance's beam + 1 best extensions."""

    def __init__(self, lp, n_frames, beam, P, ctc_weight, lm_weight=0.0):
        self.lp, self.n_frames = lp.double(), [int(n) for n in n_frames]
        self.B, self.beam, self.P, self.w, self.lm_weight = lp.shape[0], beam, P, float(ctc_weight), float(lm_weight)
        N = self.B * beam
        self.preds = torch.full((N, 1), EOS, dtype=torch.int64)
        self.scores = torch.tensor([0.0] + [NEG_INF] * (beam - 1), dtype=F64).repeat(self.B).unsqueeze(1)
        self.flag = torch.zeros(N, 1, dtype=torch.bool)
        self.state = [empty_prefix(self.lp[n // beam], self.n_frames[n // beam]) for n in range(N)]
        self.cand = self.cand_state = self.joint = None

    def joint_scores(self, att_logp, lm_logp=None):
        """-> joint f64 [N, V], -inf outside each row's P candidates; keeps the candidates and their states."""
        att = att_logp.double()
        lm = self.lm_weight * lm_logp.double() if lm_logp is not None else torch.zeros_like(att)
        base = att + lm
        N, V = base.shape
        top = base.topk(min(self.P + 1, V), dim=1)
        self.cand = top.indices[:, :self.P]
        self.prune_margin = top.values[:, self.P - 1] - top.values[:, self.P] if V > self.P else torch.full((N,), float('inf'))
        joint = torch.full((N, V), NEG_INF, dtype=F64)
        self.cand_state = []
        for n in range(N):
            c = self.cand[n]
            if self.w == 0.0:                 # no CTC term: today's search on the pre-pruned list
                joint[n, c] = base[n, c]
                self.cand_state.append(None)
                continue
            u = n // self.beam
            gamma, psi = self.state[n]
            empty = self.preds.shape[1] == 1
            g, p = extend(self.lp[u], self.n_frames[u], gamma, empty, int(self.preds[n, -1]), c)
            d = torch.where(torch.isneginf(p), p, p - psi)
            joint[n, c] = torch.where(torch.isneginf(d), d, (1.0 - self.w) * att[n, c] + self.w * d + lm[n, c])
            self.cand_state.append((g, p))
        self.joint = joint
        return joint

    def step(self, att_logp, lm_logp=None):
        joint = self.joint_scores(att_logp, lm_logp)
        N, beam = joint.shape[0], self.beam
        old_state, old_flag, old_scores = self.state, self.flag.view(-1).clone(), self.scores.clone()
        # ---- margins: per row that can still win, then among each utterance's beam + 1 best extensions
        k = joint.topk(min(beam + 1, joint.shape[1]), dim=1).values
        margin = float('inf')
        for n in torch.nonzero(~old_flag & torch.isfinite(old_scores.view(-1))).view(-1).tolist():
            margin = min(margin, float(self.prune_margin[n]), _gap(k[n, beam - 1:beam + 1]))
        fin, col = old_flag.view(N, 1), torch.arange(beam).view(1, beam)
        kk = torch.where(fin, torch.where(col == 0, 0.0, NEG_INF).to(F64).expand(N, beam), k[:, :beam])
        ext = (old_scores + kk).view(self.B, beam * beam)
        top = ext.topk(min(beam + 1, beam * beam), dim=1).values
        for u in range(self.B):
            margin = min(margin, _gap(top[u]))
        # ---- the step itself, then each surviving row takes its (parent, token)'s candidate state
        trace = []
        self.preds, self.scores, self.flag = beam_step(joint, self.preds, self.scores, self.flag, beam, trace=trace)
        parent, tok = trace[0]['parent'], trace[0]['tok']
        new_state = []
        for nn in range(N):
            p, c = int(parent[nn]), int(tok[nn])
            if c == EOS or old_flag[p] or self.cand_state[p] is None:
                new_state.append(old_state[p])
                continue
            slot = torch.nonzero(self.cand[p] == c).view(-1)
            if slot.numel():
                g, ps = self.cand_state[p]
                new_state.append((g[int(slot[0])], ps[int(slot[0])]))
            else:                             # a -inf filler from outside the candidates: nothing starts with it
                new_state.append((torch.full_like(old_state[p][0], NEG_INF), torch.tensor(NEG_INF, dtype=F64)))
        self.state = new_state
        return margin
