"""N-best rescoring (DESIGN.md 4.10) restated in float64 -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A hypothesis y is a first-pass row cut at its first <S/E> (id 1; at its length first for a CTC row); the scored sequence is
y <S/E>, teacher-forced on BOS y.  A model's second-pass score is the plain sum of its token log-probs
log_softmax(logits)[t, y'_t] over the n + 1 positions; s = s1 + weight * (sum over the models).  Per utterance: a
hypothesis equal to one ranked better by the first pass is dropped (last, score -inf); the others rank by descending s, ties
in first-pass order; the first nbest are returned.  The second-pass models are the oracle's decoder
(oracle/speech_model.py) and the LM restatements of tests/transformer_lm_ref.py and tests/rnnlm_ref.py.
"""
import torch

from oracle import speech_model as om
from tests.rnnlm_ref import rnn_lm_logits
from tests.transformer_lm_ref import transformer_lm_logits

EOS = BOS = 1
PAD = 0
NEG_INF = float('-inf')


def cut(row, length=None):
    """First-pass id row -> the hypothesis y (a list): the row up to `length`, then up to its first <S/E>."""
    row = [int(v) for v in row][:length]
    return row[:row.index(EOS)] if EOS in row else row


def token_logprobs(logits, y):
    """logits [>= n + 1, V] of the teacher-forced positions BOS y -> float64 log-probs [n + 1] of y <S/E>."""
    tgt = torch.tensor(list(y) + [EOS])
    return torch.log_softmax(logits[:len(tgt)].double(), dim=-1)[torch.arange(len(tgt)), tgt]


def combine(s1, tok_lps, weight, dtype=torch.float64):
    """s = s1 + weight * sum over the models of the sum of their token log-probs, each sum left to right in `dtype` (float32
    reproduces the kernel's additions one for one)."""
    total = torch.zeros((), dtype=dtype)
    for tl in tok_lps:
        sm = torch.zeros((), dtype=dtype)
        for v in torch.as_tensor(tl).to(dtype):
            sm = sm + v
        total = total + sm
    return torch.as_tensor(s1, dtype=dtype) + torch.as_tensor(weight, dtype=dtype) * total


def rerank(hyps, s1, tok_lps, weight, nbest, dtype=torch.float64):
    """One utterance: hyps K cut hypotheses in first-pass order, s1 their first-pass scores, tok_lps[k] the per-model token
    log-prob sequences of hyps[k] <S/E>.  -> nbest (k, y, s), best first; k is None for a dropped duplicate (y [] and
    s -inf)."""
    rows = []
    for k, y in enumerate(hyps):
        dropped = any(hyps[j] == y for j in range(k))
        s = NEG_INF if dropped else float(combine(s1[k], tok_lps[k], weight, dtype))
        rows.append((dropped, -(NEG_INF if s != s else s), k, s))
    rows.sort(key=lambda r: r[:3])
    return [(None, [], NEG_INF) if d else (k, hyps[k], s) for d, _, k, s in rows[:nbest]]


def as_tensors(ranked, width, pad=EOS):
    """rerank's output -> (ids i64 [nbest, width] y then pad, lengths i64 [nbest], scores f64 [nbest])."""
    ids = torch.full((len(ranked), width), pad, dtype=torch.int64)
    for i, (_, y, _) in enumerate(ranked):
        ids[i, :len(y)] = torch.tensor(y, dtype=torch.int64)[:width]
    return ids, torch.tensor([len(y) for _, y, _ in ranked]), torch.tensor([s for _, _, s in ranked], dtype=torch.float64)


def _teacher_forced(y):
    return torch.tensor([[BOS] + list(y)])


def decoder_token_logprobs(y, memory, n_frames, sd, prefix, policy=None, **decoder_kw):
    """The attention decoder's token log-probs of y <S/E> for one utterance: memory [T, D] of which n_frames are valid;
    decoder_kw as oracle.speech_model.transformer_decoder takes them (n_blocks, n_heads, activation, normalize_before)."""
    mask = (torch.arange(memory.shape[0]) < n_frames).unsqueeze(0)
    logits = om.transformer_decoder(_teacher_forced(y), memory.unsqueeze(0), mask, sd, prefix, policy=policy, **decoder_kw)
    return token_logprobs(logits[0], y)


def transformer_lm_token_logprobs(y, sd, prefix, n_blocks, n_heads, policy=None):
    return token_logprobs(transformer_lm_logits(_teacher_forced(y), sd, prefix, n_blocks, n_heads, policy)[0], y)


def rnn_lm_token_logprobs(y, sd, prefix, num_layers, policy=None):
    """From a zero state, as the recurrent LM scores a whole sequence."""
    return token_logprobs(rnn_lm_logits(_teacher_forced(y), sd, prefix, num_layers, policy=policy)[0][0], y)
