"""The LM-fused CTC prefix beam search on the CPU -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

fused_prefix_beam_search restates otb_ctc_prefix_beam_step's search (DESIGN.md 4.19) on top of tests/ctc_ref.py's
unfused restatement: ctcdecode's search with a character-based scorer whose scorer is a neural LM.
"""
import numpy as np

from tests.ctc_ref import NEG_INF, log_add


def fused_prefix_beam_search(frames, beam, lm, lm_weight, beta, blank=0, fp32=False, trace=None):
    """frames as ctc_ref.prefix_beam_search; lm(prefix tuple) -> the LM's next-token log-probs after <S/E> + prefix (a
    sequence over V).  -> [(tokens tuple, fused log(p_b + p_nb))] best first.

    The rules of ctc_ref.prefix_beam_search with the LM term T(c | P) = lm_weight * lm(P)[c] + beta (two separately rounded
    operations; beta alone at lm_weight 0):
      extend P_i by c:  p_nb' = ((c == last(P_i) ? p_b : tot_i) + lp(c)) + T(c | P_i);
      keep P_i, merge from its parent slot p: the extension term (frm + lp(last)) + T(last | P_p), with lm(P_p)[last]
                        as it was stored when P_i was created; the p_b path and the p_nb repeat add nothing.
    No end-of-sentence term.  fp32=True: float32 arithmetic as the kernel does.  trace (a list): each frame's
    [(prefix, extended)] per slot is appended."""
    num = np.float32 if fp32 else float

    def term(lml):
        return num(beta) if lm_weight == 0 else num(num(lm_weight) * num(lml)) + num(beta)

    cur = [((), num(0.0), num(NEG_INF), num(0.0))]          # (prefix, p_b, p_nb, stored LM log-prob of its last token)
    for cands in frames:
        lp = {}
        for c, v in cands:
            lp.setdefault(int(c), num(v))
        S = len(cands) + 1
        slot = {P: i for i, (P, _, _, _) in enumerate(cur)}
        scored = []
        blank_lp = lp.get(blank, num(NEG_INF))
        for i, (P, pb, pnb, lml) in enumerate(cur):
            tot = log_add(pb, pnb)
            last = P[-1] if P else -1
            rep = lp.get(last, num(NEG_INF))
            npb = tot + blank_lp if blank_lp != NEG_INF else num(NEG_INF)
            npnb = pnb + rep if (rep != NEG_INF and pnb != NEG_INF) else num(NEG_INF)
            if P and P[:-1] in slot and rep != NEG_INF:
                Pp, ppb, ppnb, _ = cur[slot[P[:-1]]]
                frm = ppb if (Pp[-1] if Pp else -1) == last else log_add(ppb, ppnb)
                if frm != NEG_INF:
                    npnb = log_add(npnb, (frm + rep) + term(lml))
            scored.append((log_add(npb, npnb), i * S, P, npb, npnb, lml))
            row = lm(P) if lm_weight != 0 else None
            for r, (c, v) in enumerate(cands):
                c = int(c)
                if c == blank or c < 0 or P + (c,) in slot:
                    continue
                frm = pb if c == last else tot
                sc = num(NEG_INF)
                c_lm = num(row[c]) if row is not None else num(0.0)
                if frm != NEG_INF:
                    sc = (frm + num(v)) + term(c_lm)
                scored.append((sc, i * S + 1 + r, P + (c,), num(NEG_INF), sc, c_lm))
        scored = sorted((s for s in scored if s[0] != NEG_INF), key=lambda s: (-s[0], s[1]))
        cur = [(P, pb, pnb, lml) for _, _, P, pb, pnb, lml in scored[:beam]]
        if trace is not None:
            trace.append([(P, j % S != 0) for _, j, P, _, _, _ in scored[:beam]])
    return [(P, float(log_add(pb, pnb))) for P, pb, pnb, _ in cur]
