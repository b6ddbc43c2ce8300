"""The batched beam step with a defined tie order  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

oracle.beam_search.beam_step / beam_finalize restated with one difference: every ranking orders by
(value descending, index ascending) through a stable sort, where the oracle's torch.topk / torch.sort leave the order of
equal values undefined.  That is the rule both CUDA decode paths promise (`better` / `warp_best` in
csrc/beam_common.cuh: ties -> lower index), so on rows with exact ties this restatement is the bit-exact target and the
oracle is not.  Entries equal to -inf keep their real indices and are ranked like any other value.  Finished-hypothesis
masking, the fp32 score additions and the gathers are the oracle's, step for step.
"""
import torch

from oracle.speech_model import EOS


def topk_low_index(x, k):
    """top-k along the last dimension ranked by (value descending, index ascending) -> (values, indices i64)."""
    v, i = torch.sort(x, dim=-1, descending=True, stable=True)
    return v[..., :k], i[..., :k]


def beam_step(log_probs, preds, scores, flag, beam, lm_log_probs=None, lm_weight=0.0, trace=None):
    """oracle.beam_search.beam_step with both top-k selections tie-exact (lower index first)."""
    n = scores.shape[0]
    b = n // beam
    if lm_log_probs is not None:
        log_probs = log_probs + lm_weight * lm_log_probs
    k_scores, k_tok = topk_low_index(log_probs, beam)
    fin = flag.view(n, 1)
    col = torch.arange(beam).view(1, beam)
    k_scores = torch.where(fin & (col > 0), torch.full_like(k_scores, float('-inf')), k_scores)
    k_scores = torch.where(fin & (col == 0), torch.zeros_like(k_scores), k_scores)
    k_tok = torch.where(fin.expand(n, beam), torch.full_like(k_tok, EOS), k_tok)
    cand = (scores + k_scores).view(b, beam * beam)
    new_scores, offs = topk_low_index(cand, beam)
    flat = (torch.arange(b).view(b, 1) * beam * beam + offs).view(-1)
    tok = k_tok.reshape(-1)[flat]
    parent = torch.div(flat, beam, rounding_mode='floor')
    new_preds = torch.cat((preds[parent], tok.view(-1, 1)), dim=1)
    new_flag = (new_preds[:, -1] == EOS).view(-1, 1)
    if trace is not None:
        trace.append({'k_tok': k_tok.clone(), 'offs': offs.clone(), 'parent': parent.clone(),
                      'tok': tok.clone(), 'scores': new_scores.reshape(-1).clone()})
    return new_preds, new_scores.reshape(-1, 1), new_flag


def beam_finalize(preds, scores, beam, nbest, penalty, lamda):
    """oracle.beam_search.beam_finalize with the final sort tie-exact (equal scores keep the lower hypothesis first)."""
    n = preds.shape[0]
    b = n // beam
    scores = scores.view(b, beam).clone()
    p = preds.view(b, beam, -1)
    lengths = torch.sum(torch.ne(p, EOS).float(), dim=-1)
    if penalty:
        scores = scores / torch.pow((lamda + lengths) / (lamda + 1), penalty)
    s_scores, order = torch.sort(scores, dim=-1, descending=True, stable=True)
    idx = (order + torch.arange(b).view(b, 1) * beam).view(-1)
    s_preds = preds[idx].view(b, beam, -1)
    k = min(beam, nbest)
    return s_preds[:, :k, 1:], s_scores[:, :k]
