"""TransformerLanguageModel training (model/lm.py:94-141) on top of oracle/speech_model.py -- TEST INFRASTRUCTURE, NOT PRODUCT
CODE.

The loss of the reference's Transformer LM in train(): embedding -> x * sqrt(d) + PE -> post-norm GLU encoder layers under the
causal tril mask (get_seq_mask, lm.py:14-18: no key-padding mask) -> output_project (tied to the embedding with
share_embedding) -> label-smoothed CE with PAD ignored; and its gradients through autograd.  It is the oracle's
transformer_lm_log_probs up to the logits, so policy='bf16' rounds where the CUDA path stores bf16, and residual dropout goes
through the oracle's replay hook (oracle.speech_model.set_dropout) at sites (prefix + 'blocks.i', k), k = 0 after the
self-attention and 1 after the feed-forward.  tests/golden/live_ref_transformer_lm.pt pins it to the reference's own module
(tests/test_transformer_lm_ref.py).  The optimizer update is oracle/train_step.py's clip_and_adam / transformer_lr.
"""
import torch

from oracle import speech_model as om


def transformer_lm_logits(inputs, sd, prefix, n_blocks, n_heads, policy=None):
    """inputs i64 [N, L] -> logits [N, L, V] of TransformerLanguageModel.forward (lm.py:126-138)."""
    x = om._r(sd[prefix + 'embedding.weight'], policy)[inputs]
    x, _ = om.abs_posenc(x)
    x = om._r(x, policy)
    N, L = inputs.shape
    causal = torch.tril(torch.ones(L, L)).bool().unsqueeze(0).expand(N, L, L)
    for i in range(n_blocks):
        x = om.transformer_encoder_layer(x, causal, None, sd, f'{prefix}blocks.{i}', n_heads, 'glu', False, False, policy)
    out_w = sd.get(prefix + 'output_project.weight', sd[prefix + 'embedding.weight'])
    return om._r(x, policy) @ om._r(out_w, policy).t() + sd[prefix + 'output_project.bias']


def transformer_lm_loss(inputs, targets, sd, prefix, params, policy=None):
    """TransformerLanguageModel.forward (lm.py:126-141): label-smoothed CE of the logits, PAD ignored."""
    logits = transformer_lm_logits(inputs, sd, prefix, params['num_blocks'], params['n_heads'], policy)
    return om.label_smoothing_loss(logits, targets, params['smoothing'])


def transformer_lm_loss_and_grads(inputs, targets, sd, params, policy=None):
    """loss.backward() through autograd -> (loss, {name: grad}) with the reference's names; a tied output_project.weight
    (lm.py:120-121) contributes to 'embedding.weight' and has no entry of its own."""
    leaf = {k: v.detach().clone().float().requires_grad_(True) for k, v in sd.items()}
    if params['share_embedding']:
        leaf.pop('output_project.weight', None)
    loss = transformer_lm_loss(inputs, targets, leaf, '', params, policy=policy)
    loss.backward()
    return loss.detach(), {k: v.grad if v.grad is not None else torch.zeros_like(v) for k, v in leaf.items()}
