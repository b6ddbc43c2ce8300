"""Training step of the speech transformer on the CUDA path (SURVEY.md 8a rows 16-17, 8e).

Mirror of the inner step of otrans/train/trainer.py:206-234 for `SpeechToText` (model/speech2text.py:39-64):

    loss, _ = model(inputs, targets); loss.backward(); clip_grad_norm_(params, 5); scheduler.step(); optimizer.step()

The reference differentiates its forward through torch autograd.  Here the backward is written by hand as a reverse
walk over a tape of saved bf16 activations, so that every contraction runs on the wgmma kernels (dgrad = otb_linear
with the transposed weight, residual gradients fused into its epilogue; wgrad = otb_linear_wgrad; attention backward =
otb_attention_bwd) and everything else on the HBM-bound backward kernels (csrc/backward.cu).

How a model plugs into training -- three methods on its class, and nothing here asks which class it is:

    model.train_pass(*batch, want_grads=True, grad_sink=None, grad_scale=1.0, bf16_of=None, drop_seed=None)
        -> (loss 0-d f32, {parameter name -> fp32 gradient} or None without want_grads)
    model.train_batch(*step arguments) -> batch       FusedTrainer.step's arguments, validated, as train_pass takes them
                                                      (not on a model check_fused_trainer always refuses)
    model.check_fused_trainer()                       what FusedTrainer refuses at construction, before any device work
    model.mix_batch(*batch, seed=, step=, scale=, lam=) -> (batch of pass 1, batch of pass 2)
                                                      MixSpeech's two half-batches (mixspeech_halves; speech models only)

batch is (inputs, mask, truth, truth_length or None) for a SpeechToText (forward_backward), a CTCModel
(ctc_forward_backward) and a TransducerModel (transducer_forward_backward), (inputs, targets) for the language models (lm.py).  grad_sink: name -> fp32 tensor the gradients
(x grad_scale) are ADDED into (a gradient accumulation buffer); grad_scale: a float, or an f32 0-d device tensor that the
kernels making the loss gradient read on the device (MixSpeech's lambda / accum_steps); bf16_of: see LayerPack; drop_seed: int32 device tensor [1],
the dropout seed of THIS pass (read on the device), required when a dropout rate is non-zero.  The only torch autograd node is `_TrainingLoss` (loss_with_grad), which
makes `model(inputs, targets)[0].backward()` populate `.grad` of the fp32 master parameters exactly like the reference
module; loss_train_mode is the same pass without gradients, and FusedTrainer's micro-step is train_pass into its grad_sink.

Scope: the shipped Speech-Transformer configuration -- conv front end (any kernel and stride its kernels take, with or
without front_end_layer_norm; its dropout must be 0), post- or pre-norm Transformer encoder / decoder with any of the
reference's feed-forward activations (glu, relu, gelu, tanh, swish), tied or untied output layer, `residual_dropout` as
shipped (0.1: counter-based masks in the residual GEMM's epilogue, replayed in the backward; csrc/dropout.cuh) and the
attention's output dropout (`slf_attn_dropout`, the decoder's `src_attn_dropout`: a second mask in the same epilogue);
ffn_dropout and pos_dropout must be 0 (as shipped) and raise otherwise.  The encoder may also be the shipped Conformer
layout with 64-wide heads (macaron feed-forward, rel-pos attention, then the convolution module with training-mode
BatchNorm; encoder/conformer.py:75-89).
The front end is not written here: its forward is the one recognition runs (modules.encoder_input_bf16, which also fuses
the encoder's positional input), told to keep what the backward reads, and its backward sits beside it on its class
(ConvFrontEnd.backward, ...).
The CTC-only model (model/ctc.py) is the front-end + encoder half (_encoder_fwd / _encoder_bwd) with the CTC head and
otb_ctc_loss in place of the decoder; the Transformer language model is the encoder layer (enc_layer_fwd / enc_layer_bwd)
under the causal mask.  All four models share the vocabulary head (head_fwd / head_bwd) and embedding_bwd.
"""
import math
from collections import namedtuple

import torch

from . import ops
from . import modules
from .dp import allreduce_mean_, broadcast_from_first_, rank_in
from .graphs import CapturedStep, lru_get
from .modules import ConcatFeatureFrontEnd, ConformerEncoder, ConvFrontEnd, TransformerDecoder, TransformerEncoder
from .ops import BF16, EPI_BIAS, EPI_RESID, EPI_RELU


def _bf(t):
    return t.detach().to(BF16).contiguous()


def _f(t):
    return t.detach().float().contiguous()


Lin = namedtuple('Lin', 'w wt b wname bname')      # W [N,K], W^T [K,N], fp32 bias, the names of the two parameters
_Norm = namedtuple('_Norm', 'g b name')


class LayerPack:
    """bf16 operands of the layers of one training step: W [N,K] for the forward / wgrad, W^T [K,N] for the dgrad GEMMs,
    named by their module's qualified name in `model`.  `bf16_of(param)` (optional) returns a bf16 copy of a parameter
    without a per-tensor cast kernel (FusedTrainer casts its flat fp32 master buffer once per step and hands out views)."""

    def __init__(self, model, bf16_of=None):
        self._bf16_of = bf16_of
        self._names = {m: n for n, m in model.named_modules()}

    def w(self, param):
        return self._bf16_of(param) if self._bf16_of is not None else _bf(param)

    def _lin(self, lin):
        w, name = self.w(lin.weight), self._names[lin]
        return Lin(w, w.t().contiguous(), _f(lin.bias), name + '.weight', name + '.bias')

    def _ln(self, norm):
        return _Norm(_f(norm.weight), _f(norm.bias), self._names[norm])

    def enc_layer(self, b):
        a, f = b.slf_attn, b.feed_forward
        return {'qkv': self._lin(a.qvk_proj), 'o': self._lin(a.output_proj), 'w1': self._lin(f.w_1), 'w2': self._lin(f.w_2),
                'ln1': self._ln(b.norm1), 'ln2': self._ln(b.norm2), 'act': f.activation}


def check_heads(name, d_model, blocks):
    """The attention backward (otb_attention_bwd) is written for 64-wide heads: refuse any other width in the stack `name`."""
    for blk in blocks:
        if d_model != 64 * blk.n_heads:
            raise NotImplementedError(f'training path: 64-wide attention heads only; the {name} has d_model {d_model} '
                                      f'with {blk.n_heads} heads')


_ATTN_DROPOUT = ('slf_attn_dropout', 'src_attn_dropout')


def check_blocks(blocks):
    """The feed-forward and dropout rules of a stack of blocks -> the residual_dropout rate of every block (the attention
    output's rates: attn_dropout_rates)."""
    out = []
    for blk in blocks:
        if _ffn_of(blk).activation not in ('glu', 'relu') + tuple(ops.TRAIN_ACT):
            raise NotImplementedError(f'training path: feed-forward activation {_ffn_of(blk).activation!r}')
        rates = getattr(blk, 'dropout_rates', {})
        # conv_dropout: the reference builds the Dropout and never applies it (module/conformer.py:34,36-57)
        other = {k: v for k, v in rates.items() if k not in ('residual_dropout', 'conv_dropout') + _ATTN_DROPOUT and float(v) > 0.0}
        if other:
            # the reference applies these in train mode (ffn.py:40, pos.py); training WITHOUT them would be a different
            # network, so refuse instead of silently dropping the regulariser.  residual_dropout and the attention output's
            # dropout ARE implemented (otb_linear_dropout_resid / otb_dropout_bwd).
            raise NotImplementedError(f'training path: only residual_dropout and the attention dropout are implemented, got '
                                      f'{other}; set them to 0.0')
        for k in ('residual_dropout',) + _ATTN_DROPOUT:
            if not (0.0 <= float(rates.get(k, 0.0)) < 1.0):
                raise ValueError(f'{k} must be in [0, 1)')
        out.append(float(rates.get('residual_dropout', 0.0)))
    return out


def attn_dropout_rates(blk):
    """The attention-output dropout rate of each residual sub-layer of a block, in site order (attention.py:46: the
    attention returns dropout(output_proj(context)), and the layer's residual dropout lands on top): a Transformer encoder
    layer (slf_attn_dropout, 0 for the feed-forward), a decoder layer (slf_attn_dropout, src_attn_dropout, 0).  A
    Conformer's rel-pos attention takes none (its constructor refuses a rate)."""
    rates = getattr(blk, 'dropout_rates', {})
    slf, src = float(rates.get('slf_attn_dropout', 0.0)), float(rates.get('src_attn_dropout', 0.0))
    if hasattr(blk, 'src_attn'):
        return (slf, src, 0.0)
    return (0.0, 0.0, 0.0) if hasattr(blk, 'pre_ffn') else (slf, 0.0)


def _flat(per_block):
    return [r for rates in per_block for r in rates]


def need_drop_seed(drop_seed, rates):
    if drop_seed is None and any(r > 0.0 for r in rates):
        raise ValueError('training pass: a dropout rate > 0 needs a drop_seed tensor')


class EncoderPack(LayerPack):
    """The LayerPack of the front end and the encoder: all a CTCModel trains, and the first half of a SpeechToText's
    TrainPack.  Its constructor refuses what the training path does not cover, before any device work.  Where the model
    has a decoder the checks take it in beside the encoder, each rule over both stacks before the next rule, so that the
    refusal a configuration with two faults gets does not depend on the stack a fault sits in (96-wide decoder heads and a
    320-channel front end: the heads).  `rates`: stack name -> the residual_dropout rate of every block; `attn_rates`: stack
    name -> attn_dropout_rates of every block."""

    def __init__(self, model, bf16_of=None, with_decoder=True):
        super().__init__(model, bf16_of)
        # with_decoder False: the model's `decoder` is no attention stack (a transducer's prediction network)
        fe, enc = model.frontend, model.encoder
        dec = getattr(model, 'decoder', None) if with_decoder else None
        self.conformer = isinstance(enc, ConformerEncoder)
        if not (isinstance(fe, (ConvFrontEnd, ConcatFeatureFrontEnd)) and isinstance(enc, (TransformerEncoder, ConformerEncoder))
                and (dec is None or isinstance(dec, TransformerDecoder))):
            raise NotImplementedError('training path: conv or concat front end + Transformer or Conformer encoder'
                                      + (' + Transformer decoder' if dec is not None else '') + ' only')
        if not self.conformer and enc.relative_positional:
            raise NotImplementedError('training path: the Transformer encoder with absolute positions only')
        stacks = [('encoder', enc)] + ([('decoder', dec)] if dec is not None else [])
        for name, stack in stacks:
            check_heads(name, stack.d_model, stack.blocks)
        if isinstance(fe, ConvFrontEnd):
            C1 = fe.conv1.conv_layer.out_channels
            if (C1 + 63) // 64 * 64 > 256:       # the conv1 weight gradient (otb_conv1_wgrad) runs one channel per thread
                raise NotImplementedError(f'training path: mid_channel {C1} pads to {(C1 + 63) // 64 * 64} channels; the conv1 '
                                          'weight gradient takes at most 256')
            if fe.dropout > 0.0:
                raise NotImplementedError(f'training path: front-end dropout {fe.dropout} is not implemented; set it to 0.0')
            if fe.front_end_layer_norm and (fe.output_size > 256 or fe.output_size % 8):
                raise NotImplementedError(f'training path: front_end_layer_norm over output_size {fe.output_size}; its '
                                          'backward (otb_layernorm_bwd) takes a multiple of 8, at most 256')
        if self.conformer:
            _check_conformer(enc)
        if any(stack.pos_emb.scale_learnable for _, stack in stacks):
            raise NotImplementedError('training path: learnable positional scale (pos_dropout > 0)')
        self.rates = {name: check_blocks(stack.blocks) for name, stack in stacks}
        self.attn_rates = {name: [attn_dropout_rates(b) for b in stack.blocks] for name, stack in stacks}
        self.fe = fe.training_pack(self.w)
        self.enc = [self._conf_layer(b) if self.conformer else self.enc_layer(b) for b in enc.blocks]
        # pre-norm stacks end with one more LayerNorm (encoder/transformer.py:96-97,131-132; decoder/transformer.py:151-152,178-179)
        self.enc_pre = bool(getattr(enc, 'normalize_before', False))
        self.enc_norm = self._ln(enc.norm) if self.enc_pre else None

    def _conf_layer(self, b):
        """A Conformer block: the rel-pos projection as ONE GEMM producing [q+u | q+v | k | v] (W_ext = [Wq; Wq; Wk; Wv],
        b_ext = [bq + u; bq + v; bk; bv], as the inference pack), and the convolution module with BatchNorm unfolded."""
        a, cv = b.mha, b.conv
        w = self.w(a.qvk_proj.weight)
        d = w.shape[1]
        wext = torch.cat([w[:d], w], 0)
        bq = _f(a.qvk_proj.bias)
        bext = torch.cat([bq[:d] + _f(a.posu).reshape(d), bq[:d] + _f(a.posv).reshape(d), bq[d:]])
        dw, bn = cv.depthwise_conv, cv.batch_norm
        return {'mac_ln': self._ln(b.macaron_ffn_norm), 'w1': self._lin(b.pre_ffn.w_1), 'w2': self._lin(b.pre_ffn.w_2),
                'act': b.pre_ffn.activation, 'scale': float(b.ffn_scale),
                'mha_ln': self._ln(b.mha_norm), 'wext': wext, 'wext_t': wext.t().contiguous(), 'bext': bext,
                'wpos': self.w(a.pos_proj.weight), 'attn': self._names[a],
                'conv_ln': self._ln(b.conv_norm), 'pw1': self._lin(cv.pointwise_conv1), 'pw2': self._lin(cv.pointwise_conv2),
                'dw': _f(dw.weight).view(d, -1), 'dwb': _f(dw.bias), 'dw_name': self._names[dw],
                'bn': bn, 'bn_g': _f(bn.weight), 'bn_b': _f(bn.bias), 'bn_name': self._names[bn],
                'post_ln': self._ln(b.post_ffn_norm), 'final_ln': self._ln(b.final_norm)}


class TrainPack(EncoderPack):
    """The LayerPack of a SpeechToText model: front end, encoder and decoder layers and the output layer."""

    def __init__(self, model, bf16_of=None):
        super().__init__(model, bf16_of)
        dec = model.decoder
        self.dec = [self._dec_layer(b) for b in dec.blocks]
        self.dec_pre = bool(dec.normalize_before)
        self.dec_norm = self._ln(dec.after_norm) if self.dec_pre else None
        self.emb = self.w(dec.embedding.weight)
        # the output layer's weight gradient goes by the embedding's name when the two are one tensor
        tied = dec.output_layer.weight is dec.embedding.weight
        self.wout = self.emb if tied else self.w(dec.output_layer.weight)
        self.wout_name = 'decoder.embedding.weight' if tied else 'decoder.output_layer.weight'
        self.bout = _f(dec.output_layer.bias)

    def _dec_layer(self, b):
        a, c, f = b.slf_attn, b.src_attn, b.feed_forward
        return {'qkv': self._lin(a.qvk_proj), 'o': self._lin(a.output_proj), 'q': self._lin(c.q_proj),
                'kv': self._lin(c.vk_proj), 'o2': self._lin(c.output_proj), 'w1': self._lin(f.w_1), 'w2': self._lin(f.w_2),
                'ln1': self._ln(b.norm1), 'ln2': self._ln(b.norm2), 'ln3': self._ln(b.norm3), 'act': f.activation}


def _ffn_of(blk):
    return blk.pre_ffn if hasattr(blk, 'pre_ffn') else blk.feed_forward


def _check_conformer(enc):
    """The Conformer layout the training path builds: the reference's shipped block (conformer_baseline.yaml)."""
    if not (enc.positional_encoding and enc.relative_positional):
        raise NotImplementedError('training path: the Conformer with relative positional encoding only '
                                  '(positional_encoding and relative_positional True)')
    for blk in enc.blocks:
        if not blk.macaron_style or blk.conv_first:
            raise NotImplementedError('training path: the Conformer block with macaron_style True and conv_first False only')
        if not blk.conv_bias:
            raise NotImplementedError('training path: the Conformer convolution module with conv_bias True only')
        bn = blk.conv.batch_norm
        if bn.momentum is None or not bn.track_running_stats or not bn.affine:
            raise NotImplementedError('training path: BatchNorm1d with momentum, running statistics and affine parameters')


def unused_parameters(model):
    """Names of the parameters the forward never reads: a Conformer block's post_ffn (the reference applies only
    post_ffn_norm, encoder/conformer.py:87-89), so their .grad stays None and the optimizer never moves them.  A model
    without an encoder (a language model) reads all of its parameters."""
    if not isinstance(getattr(model, 'encoder', None), ConformerEncoder):
        return set()
    return {n for n, _ in model.named_parameters() if '.post_ffn.' in n and n.startswith('encoder.blocks.')}


class Grads(dict):
    """name -> fp32 gradient.  With `sink` (name -> fp32 view of the optimizer's flat gradient buffer) the kernels ADD
    their result straight into the sink (otb_linear_wgrad / otb_colsum / otb_layernorm_bwd accumulate flags) -- what
    autograd's AccumulateGrad does, without one torch add per parameter."""

    def __init__(self, sink=None):
        super().__init__()
        self.sink = sink

    def out(self, name):
        return self.sink[name] if self.sink is not None else None

    def put(self, name, value):
        """For gradients produced by code that cannot accumulate in place."""
        if self.sink is not None:
            self.sink[name].add_(value.reshape(self.sink[name].shape))
            self[name] = self.sink[name]
        else:
            self[name] = value.contiguous()


def _norm(x, ln):
    return ops.layernorm(x, ln.g, ln.b)


def _ln_bwd(dy, z, ln, grads):
    acc = grads.sink is not None
    wname, bname = ln.name + '.weight', ln.name + '.bias'
    dz, dg, db = ops.layernorm_bwd(dy, z, ln.g, dgamma=grads.out(wname), dbeta=grads.out(bname), accumulate=acc)
    grads[wname], grads[bname] = dg, db
    return dz


def linear_bwd(dy, x, lin, grads, resid=None):
    """Gradients of y = x W^T + b: parameter grads into `grads`, returns dx (+ resid) as bf16."""
    acc = grads.sink is not None
    grads[lin.wname] = ops.linear_wgrad(dy, x, out=grads.out(lin.wname), accumulate=acc)
    grads[lin.bname] = ops.colsum(dy, out=grads.out(lin.bname), accumulate=acc)
    if resid is not None:
        return ops.linear(dy, lin.wt, None, EPI_RESID, resid=resid)
    return ops.linear(dy, lin.wt)


# dropout site ids: Transformer encoder layer i -> 2 i + {0, 1}; Conformer block i -> 3 i + {0, 1, 2} (macaron feed-forward,
# attention, convolution module); decoder layer i -> 1000 + 3 i + {0, 1, 2}; the same decoder layer in the MWER branch,
# over the n-best (forward_backward's nbest) -> 4000 + 3 i + {0, 1, 2}, clear of the language models' 2000 + / 3000 + (lm.py).
# The attention-output mask of the sub-layer whose residual mask is site s is site ATTN_SITE + s: every residual range
# above moved up by 5000, clear of all of them, so that turning the attention dropout on draws the same residual masks.
ENC_SITE, DEC_SITE, MWER_SITE = 0, 1000, 4000
ATTN_SITE = 5000


def _enc_sites(enc):
    return 3 if isinstance(enc, ConformerEncoder) else 2


def _ffn_fwd(p, x):
    """First half of the position-wise feed-forward (ffn.py:38-41): returns (pre-activation u or None, hidden h)."""
    if p['act'] == 'relu':
        return None, ops.linear(x, p['w1'].w, p['w1'].b, EPI_RELU)  # ReLU fused into the GEMM; its backward needs only h
    u = ops.linear(x, p['w1'].w, p['w1'].b)
    return u, (ops.glu_fwd(u) if p['act'] == 'glu' else ops.act_fwd(u, p['act']))


def _ffn_act_bwd(p, dh, u, h):
    if p['act'] == 'relu':
        return ops.relu_bwd(dh, h)
    return ops.glu_bwd(dh, u) if p['act'] == 'glu' else ops.act_bwd(dh, u, p['act'])


def dropout_sites(model):
    """[(site id, 'encoder' | 'decoder', rate)] of every residual-dropout site (what a parity test must replay; the
    attention-output sites: attn_dropout_sites)."""
    out = []
    n = _enc_sites(model.encoder)
    for i, b in enumerate(model.encoder.blocks):
        out += [(ENC_SITE + n * i + k, 'encoder', float(b.dropout_rates['residual_dropout'])) for k in range(n)]
    for i, b in enumerate(model.decoder.blocks if getattr(model, 'decoder', None) is not None else []):
        out += [(DEC_SITE + 3 * i + k, 'decoder', float(b.dropout_rates['residual_dropout'])) for k in range(3)]
    return out


def attn_dropout_sites(model):
    """[(site id, 'encoder' | 'decoder', rate)] of every attention-output dropout site with a non-zero rate: the sub-layer
    whose residual site is s draws its attention mask at ATTN_SITE + s (both masks on the same tensor)."""
    out = []
    n = _enc_sites(model.encoder)
    for i, b in enumerate(model.encoder.blocks):
        out += [(ATTN_SITE + ENC_SITE + n * i + k, 'encoder', r) for k, r in enumerate(attn_dropout_rates(b)) if r > 0.0]
    for i, b in enumerate(model.decoder.blocks if getattr(model, 'decoder', None) is not None else []):
        out += [(ATTN_SITE + DEC_SITE + 3 * i + k, 'decoder', r) for k, r in enumerate(attn_dropout_rates(b)) if r > 0.0]
    return out


def _drops(rates, attn_rates, seed, site0, per_layer):
    """The `drop` of every layer of a stack: (residual rate, seed tensor, site id of the layer's sub-layer 0, attention-output
    rate of each sub-layer)."""
    return [(r, seed, site0 + per_layer * i, a) for i, (r, a) in enumerate(zip(rates, attn_rates))]


def _attn_rate(drop, k):
    """The attention-output dropout rate of sub-layer k; a drop of three (the language models') carries none."""
    return drop[3][k] if len(drop) > 3 else 0.0


def _resid(ctx, lin, x, drop, k, alpha=1.0):
    """x + alpha * dropout(ctx W^T + b): the residual connection of sub-layer k in training mode (transformer.py:54,61);
    with an attention-output rate, the attention's own dropout first (attention.py:46).  drop = (rate, seed tensor, site id
    of the layer's sub-layer 0[, attention-output rate of each sub-layer])."""
    rate, seed, site = drop[:3]
    pa = _attn_rate(drop, k)
    if rate > 0.0 or pa > 0.0:
        return ops.linear_dropout_resid(ctx, lin.w, lin.b, x, rate, seed, site + k, alpha=alpha, p2=pa, site2=ATTN_SITE + site + k)
    return ops.linear(ctx, lin.w, lin.b, EPI_RESID, resid=x, alpha=alpha)


def _drop_bwd(dz, drop, k):
    rate, seed, site = drop[:3]
    pa = _attn_rate(drop, k)
    return ops.dropout_bwd(dz, rate, seed, site + k, p2=pa, site2=ATTN_SITE + site + k) if rate > 0.0 or pa > 0.0 else dz


# What a layer saves for its backward.  Sub-layer k has input u_k and residual sum z_k = u_k + drop(f_k(u_k)).  Pre-norm
# (the reference takes the residual AFTER the norm): u_1 = norm1(a), u_k+1 = norm_k+1(z_k), the output is z_last.
# Post-norm: u_1 = a, u_k+1 = norm_k(z_k), the output is norm_last(z_last).  a is the layer input; ffn_u is the feed-forward's
# pre-activation (None with ReLU, whose backward reads h) and h its hidden activation.
_EncTape = namedtuple('_EncTape', 'a u1 qkv ctx lse z1 u2 ffn_u h z2')
_DecTape = namedtuple('_DecTape', 'a u1 qkv ctx lse z1 u2 q kv ctx2 lse2 z2 u3 ffn_u h z3')


def enc_layer_fwd(p, a, pre, B, H, T, lengths, drop, causal=False):
    """One encoder layer in training mode (encoder/transformer.py:41-65) -> (output, _EncTape).  causal=True: the tril
    mask the Transformer LM feeds to the same layer (model/lm.py:14-18)."""
    d = a.shape[1]
    u1 = _norm(a, p['ln1']) if pre else a
    qkv = ops.linear(u1, p['qkv'].w, p['qkv'].b)
    ctx, lse = ops.attention_train(qkv, qkv, qkv, B, H, T, T, kv_len=lengths, causal=causal, q_col0=0, k_col0=d, v_col0=2 * d)
    z1 = _resid(ctx, p['o'], u1, drop, 0)
    u2 = _norm(z1, p['ln2'] if pre else p['ln1'])
    ffn_u, h = _ffn_fwd(p, u2)
    z2 = _resid(h, p['w2'], u2, drop, 1)
    out = z2 if pre else _norm(z2, p['ln2'])
    return out, _EncTape(a=a, u1=u1, qkv=qkv, ctx=ctx, lse=lse, z1=z1, u2=u2, ffn_u=ffn_u, h=h, z2=z2)


def enc_layer_bwd(p, t, dout, pre, g, B, H, T, lengths, drop, causal=False):
    """Backward of enc_layer_fwd: parameter gradients into g; returns the gradient of the layer input."""
    d = t.a.shape[1]
    dz2 = dout if pre else _ln_bwd(dout, t.z2, p['ln2'], g)
    # the sub-layer branch sees the replayed dropout mask, the residual branch (resid=) the plain gradient
    dh = linear_bwd(_drop_bwd(dz2, drop, 1), t.h, p['w2'], g)
    du2 = linear_bwd(_ffn_act_bwd(p, dh, t.ffn_u, t.h), t.u2, p['w1'], g, resid=dz2)
    dz1 = _ln_bwd(du2, t.z1, p['ln2'] if pre else p['ln1'], g)
    dctx = linear_bwd(_drop_bwd(dz1, drop, 0), t.ctx, p['o'], g)
    dqkv = torch.empty_like(t.qkv)
    ops.attention_bwd(t.qkv, t.qkv, t.qkv, t.ctx, dctx, t.lse, B, H, T, T, dqkv, dqkv, dqkv, kv_len=lengths, causal=causal,
                      q_col0=0, k_col0=d, v_col0=2 * d, dq_col0=0, dk_col0=d, dv_col0=2 * d)
    du1 = linear_bwd(dqkv, t.u1, p['qkv'], g, resid=dz1)
    return _ln_bwd(du1, t.a, p['ln1'], g) if pre else du1


def _dec_layer_fwd(p, a, mem, pre, B, H, L, T, lengths, drop, K=1):
    """One decoder layer in training mode (decoder/transformer.py:54-90) over the memory mem -> (output, _DecTape).
    a holds K sequences of L rows per utterance: self-attention is causal within each of the B*K sequences, and
    cross-attention treats the K*L query rows of utterance b as one problem against its memory (score_bf16's layout), so
    the memory's K|V is projected once per utterance."""
    d = a.shape[1]
    u1 = _norm(a, p['ln1']) if pre else a
    qkv = ops.linear(u1, p['qkv'].w, p['qkv'].b)
    ctx, lse = ops.attention_train(qkv, qkv, qkv, B * K, H, L, L, causal=True, q_col0=0, k_col0=d, v_col0=2 * d)
    z1 = _resid(ctx, p['o'], u1, drop, 0)
    u2 = _norm(z1, p['ln2'] if pre else p['ln1'])
    q = ops.linear(u2, p['q'].w, p['q'].b)
    kv = ops.linear(mem, p['kv'].w, p['kv'].b)
    ctx2, lse2 = ops.attention_train(q, kv, kv, B, H, K * L, T, kv_len=lengths, k_col0=0, v_col0=d)
    z2 = _resid(ctx2, p['o2'], u2, drop, 1)
    u3 = _norm(z2, p['ln3'] if pre else p['ln2'])
    ffn_u, h = _ffn_fwd(p, u3)
    z3 = _resid(h, p['w2'], u3, drop, 2)
    out = z3 if pre else _norm(z3, p['ln3'])
    return out, _DecTape(a=a, u1=u1, qkv=qkv, ctx=ctx, lse=lse, z1=z1, u2=u2, q=q, kv=kv, ctx2=ctx2, lse2=lse2, z2=z2,
                         u3=u3, ffn_u=ffn_u, h=h, z3=z3)


def _dec_layer_bwd(p, t, dout, dmem, mem, pre, g, B, H, L, T, lengths, drop, K=1):
    """Backward of _dec_layer_fwd: parameter gradients into g; returns the gradient of the layer input and dmem plus
    this layer's gradient of the memory (added by the K|V dgrad GEMM's residual epilogue), summed over the K sequences."""
    d = t.a.shape[1]
    dz3 = dout if pre else _ln_bwd(dout, t.z3, p['ln3'], g)
    dh = linear_bwd(_drop_bwd(dz3, drop, 2), t.h, p['w2'], g)
    du3 = linear_bwd(_ffn_act_bwd(p, dh, t.ffn_u, t.h), t.u3, p['w1'], g, resid=dz3)
    dz2 = _ln_bwd(du3, t.z2, p['ln3'] if pre else p['ln2'], g)
    dctx2 = linear_bwd(_drop_bwd(dz2, drop, 1), t.ctx2, p['o2'], g)
    dq = torch.empty_like(t.q)
    dkv = torch.empty_like(t.kv)
    ops.attention_bwd(t.q, t.kv, t.kv, t.ctx2, dctx2, t.lse2, B, H, K * L, T, dq, dkv, dkv, kv_len=lengths, k_col0=0, v_col0=d,
                      dq_col0=0, dk_col0=0, dv_col0=d)
    dmem = linear_bwd(dkv, mem, p['kv'], g, resid=dmem)
    du2 = linear_bwd(dq, t.u2, p['q'], g, resid=dz2)
    dz1 = _ln_bwd(du2, t.z1, p['ln2'] if pre else p['ln1'], g)
    dctx = linear_bwd(_drop_bwd(dz1, drop, 0), t.ctx, p['o'], g)
    dqkv = torch.empty_like(t.qkv)
    ops.attention_bwd(t.qkv, t.qkv, t.qkv, t.ctx, dctx, t.lse, B * K, H, L, L, dqkv, dqkv, dqkv, causal=True, q_col0=0, k_col0=d,
                      v_col0=2 * d, dq_col0=0, dk_col0=d, dv_col0=2 * d)
    du1 = linear_bwd(dqkv, t.u1, p['qkv'], g, resid=dz1)
    return (_ln_bwd(du1, t.a, p['ln1'], g) if pre else du1), dmem


# A Conformer block (encoder/conformer.py:75-89, macaron, rel-pos attention, then the convolution module):
#   x1 = x0 + ffn_scale * drop(pre_ffn(y0)),  y0 = macaron_ffn_norm(x0)          (h: activation output, ffn_u: its input)
#   x2 = x1 + drop(relmha(y1)),               y1 = mha_norm(x1)                  (ext = [q+u | q+v | k | v], pproj = pos_proj(PE))
#   x3 = x2 + drop(mask(conv(y2))),           y2 = conv_norm(x2)                 (cu: pointwise_conv1 output, g = GLU(cu),
#                                                                                 c / stats: depthwise conv and BatchNorm statistics,
#                                                                                 s = swish(BN(c)) zero on padded frames)
#   out = final_norm(z),                      z = post_ffn_norm(x3)
_ConfTape = namedtuple('_ConfTape', 'x0 y0 ffn_u h x1 y1 ext pproj ctx lse x2 y2 cu g c stats s x3 z')


def _conformer_block_fwd(p, x0, B, H, T, lengths, pe, drop):
    """One Conformer block in training mode -> (output, _ConfTape).  pe: bf16 PE[-(T-1) .. T-1]; the BatchNorm running
    statistics are updated on the device."""
    rate, seed, site = drop[:3]
    d = x0.shape[1]
    y0 = _norm(x0, p['mac_ln'])
    ffn_u, h = _ffn_fwd(p, y0)
    x1 = _resid(h, p['w2'], x0, drop, 0, alpha=p['scale'])
    y1 = _norm(x1, p['mha_ln'])
    ext = ops.linear(y1, p['wext'], p['bext'])
    pproj = ops.linear(pe, p['wpos'])
    bd = modules.rel_pos_band(ext, pproj, H, B, T)
    ctx, lse = ops.attention_train(ext, ext, ext, B, H, T, T, kv_len=lengths, q_col0=0, k_col0=2 * d, v_col0=3 * d, bd=bd)
    del bd                   # recomputed by the backward: [H, B*T, 2T] fp32 is the largest tensor of the block
    x2 = ops.dropout_add(ctx, x1, rate, seed, site + 1)
    y2 = _norm(x2, p['conv_ln'])
    cu = ops.linear(y2, p['pw1'].w, p['pw1'].b)
    g = ops.glu_fwd(cu)
    bn = p['bn']
    s, c, stats = ops.conformer_conv_train(g, lengths, p['dw'], p['dwb'], p['bn_g'], p['bn_b'], bn.running_mean, bn.running_var,
                                           bn.num_batches_tracked, B, T, momentum=bn.momentum, eps=bn.eps)
    co = ops.linear(s, p['pw2'].w, p['pw2'].b)
    x3 = ops.dropout_add(co, x2, rate, seed, site + 2, row_len=lengths, row_period=T)
    z = _norm(x3, p['post_ln'])
    return _norm(z, p['final_ln']), _ConfTape(x0=x0, y0=y0, ffn_u=ffn_u, h=h, x1=x1, y1=y1, ext=ext, pproj=pproj, ctx=ctx, lse=lse,
                                              x2=x2, y2=y2, cu=cu, g=g, c=c, stats=stats, s=s, x3=x3, z=z)


def _acc_out(g, name, shape, dev):
    """The gradient tensor of `name` that kernels ADD into: the optimizer's sink, else a fresh zero tensor."""
    out = g.out(name)
    if out is None:
        out = torch.zeros(shape, dtype=torch.float32, device=dev)
    g[name] = out
    return out


def _relpos_attn_bwd(p, t, dctx, g, B, H, T, lengths, pe):
    """Backward of the rel-pos attention (attention.py:196-253): attention with the band, the band's GEMMs, pos_proj,
    posu / posv and qvk_proj (whose q rows feed both q+u and q+v).  Returns the gradient of y1 (bf16)."""
    d = dctx.shape[1]
    dk, M, n, dev = d // H, B * T, 2 * T - 1, dctx.device
    bd = modules.rel_pos_band(t.ext, t.pproj, H, B, T)
    ldb = ops.rel_band_ld(T)
    dbd = torch.zeros(H, M, ldb, dtype=BF16, device=dev)
    de = torch.empty_like(t.ext)                                                 # d[q+u | q+v | k | v]
    ops.attention_bwd(t.ext, t.ext, t.ext, t.ctx, dctx, t.lse, B, H, T, T, de, de, de, kv_len=lengths, q_col0=0, k_col0=2 * d,
                      v_col0=3 * d, dq_col0=0, dk_col0=2 * d, dv_col0=3 * d, bd=bd, dbd=dbd)
    del bd
    pt = torch.zeros(d, ldb, dtype=BF16, device=dev)                            # P^T, zero columns up to the band pitch
    pt[:, :n] = t.pproj.t()
    dp = torch.empty(ldb, d, dtype=torch.float32, device=dev)
    for h in range(H):
        ops.linear(dbd[h], pt[dk * h: dk * (h + 1)], out=de[:, d + dk * h: d + dk * (h + 1)])       # d(q+v)_h = dBD_h P_h
        ops.linear_wgrad(dbd[h], t.ext[:, d + dk * h: d + dk * (h + 1)], out=dp[:, dk * h: dk * (h + 1)])   # dP_h = dBD_h^T (q+v)_h
    acc = g.sink is not None
    pname = p['attn'] + '.pos_proj.weight'
    g[pname] = ops.linear_wgrad(ops.scale_add_table(dp[:n]), pe, out=g.out(pname), accumulate=acc)     # dW_pos = dP^T PE
    qn = p['attn'] + '.qvk_proj'
    dw = _acc_out(g, qn + '.weight', (3 * d, d), dev)
    db = _acc_out(g, qn + '.bias', (3 * d,), dev)
    for part in (de[:, :d], de[:, d:2 * d]):        # q+u and q+v both come from the q rows
        ops.linear_wgrad(part, t.y1, out=dw[:d], accumulate=True)
        ops.colsum(part, out=db[:d], accumulate=True)
    ops.linear_wgrad(de[:, 2 * d:], t.y1, out=dw[d:], accumulate=True)
    ops.colsum(de[:, 2 * d:], out=db[d:], accumulate=True)
    for k, name in enumerate(('posu', 'posv')):
        ops.colsum(de[:, k * d:(k + 1) * d], out=_acc_out(g, p['attn'] + '.' + name, (1, 1, H, dk), dev).view(d), accumulate=True)
    return ops.linear(de, p['wext_t'])


def _conformer_block_bwd(p, t, dout, g, B, H, T, lengths, pe, drop):
    """Backward of _conformer_block_fwd: parameter gradients into g; returns the gradient of the block input."""
    rate, seed, site = drop[:3]
    acc = g.sink is not None
    dz = _ln_bwd(dout, t.z, p['final_ln'], g)
    dx3 = _ln_bwd(dz, t.x3, p['post_ln'], g)
    # convolution module: its output was masked, then dropped
    dco = ops.dropout_add(dx3, None, rate, seed, site + 2, row_len=lengths, row_period=T)
    ds = linear_bwd(dco, t.s, p['pw2'], g)
    dwn, bwn, bn = p['dw_name'] + '.weight', p['dw_name'] + '.bias', p['bn_name']
    dg, dwv, g[bwn], g[bn + '.weight'], g[bn + '.bias'] = ops.conformer_conv_bwd(
        ds, t.g, lengths, p['dw'], p['bn_g'], p['bn_b'], t.c, t.stats, B, T, dw=g.out(dwn).view(p['dw'].shape) if acc else None,
        dwb=g.out(bwn), dgamma=g.out(bn + '.weight'), dbeta=g.out(bn + '.bias'), accumulate=acc)
    g[dwn] = g.out(dwn) if acc else dwv.view(dwv.shape[0], 1, -1)             # nn.Conv1d's [d, 1, k]
    dy2 = linear_bwd(ops.glu_bwd(dg, t.cu), t.y2, p['pw1'], g)
    dx2 = ops.dropout_add(_ln_bwd(dy2, t.x2, p['conv_ln'], g), dx3)
    # rel-pos attention (no output projection)
    dy1 = _relpos_attn_bwd(p, t, _drop_bwd(dx2, drop, 1), g, B, H, T, lengths, pe)
    dx1 = ops.dropout_add(_ln_bwd(dy1, t.x1, p['mha_ln'], g), dx2)
    # macaron feed-forward, scaled by ffn_scale
    df = ops.dropout_add(dx1, None, rate, seed, site, alpha=p['scale'])
    dh = linear_bwd(df, t.h, p['w2'], g)
    dy0 = linear_bwd(_ffn_act_bwd(p, dh, t.ffn_u, t.h), t.y0, p['w1'], g)
    return ops.dropout_add(_ln_bwd(dy0, t.x0, p['mac_ln'], g), dx1)


def head_fwd(y, w, b, ld):
    """A vocabulary head, logits = y W^T + b -> f32 [rows, ld] (ld = V padded, the first V columns valid): the attention
    decoder's output layer, the CTC head and the language models' output projection."""
    return ops.linear(y, w, b, EPI_BIAS, out_f32=True, n_out=ld)


def head_bwd(dlogits, y, w, g, wname, bname, resid=None):
    """Backward of head_fwd from dlogits [rows, ld]: the gradient of W (bf16 [V, d]) into g[wname] -- the embedding's name
    when the head is tied to it, and embedding_bwd then lands on top -- and of b into g[bname].  Returns dy (+ resid) as
    bf16 [rows, d].  The zero-padded W^T of the dgrad GEMM is built here, every pass: the weights move every step."""
    V, d = w.shape
    # dlogits[:, :V] as a strided view: the TMA map stops at column V, so the result has exactly V rows
    g[wname] = ops.linear_wgrad(dlogits[:, :V], y, out=g.out(wname), accumulate=g.sink is not None)
    g.put(bname, ops.colsum(dlogits)[:V])
    wt = torch.zeros(d, dlogits.shape[1], dtype=BF16, device=w.device)
    wt[:, :V] = w.t()
    if resid is not None:
        return ops.linear(dlogits, wt, None, EPI_RESID, resid=resid)
    return ops.linear(dlogits, wt)


def embedding_bwd(tok, dx, emb, scale, g, name):
    """Backward of x = scale * E[tok] (E: emb) into g[name].  With a tied head g[name] already holds the head's gradient,
    and the embedding's lands on top of it (fp32 atomics)."""
    if name not in g:
        _acc_out(g, name, emb.shape, dx.device)
    ops.embed_bwd(tok, dx, g[name], scale)


# fe: what the front end's backward reads (its rows_bf16's saved); pe: the rel-pos table of a Conformer
_EncTrace = namedtuple('_EncTrace', 'fe tape pe lengths enc_last drops B T2')


def _encoder_fwd(model, pk, inputs, mask, drop_seed):
    """Front end + encoder in training mode, the half shared by SpeechToText, CTCModel and TransducerModel -> (memory bf16
    [B*T', d], _EncTrace: what _encoder_bwd reads).  The front half is the one recognition runs (encoder_input_bf16), on
    the training pack's front-end operands."""
    enc = model.encoder
    B = inputs.shape[0]
    H = enc.blocks[0].n_heads
    x, lengths, T2, fe_saved = modules.encoder_input_bf16(model.frontend, enc, inputs, mask, pk.fe, keep=True)
    e_drop = _drops(pk.rates['encoder'], pk.attn_rates['encoder'], drop_seed, ENC_SITE, _enc_sites(enc))
    enc_tape = []
    pe = enc.rel_pos_table(T2, inputs.device)
    for p, drop in zip(pk.enc, e_drop):
        if pk.conformer:
            x, t = _conformer_block_fwd(p, x, B, H, T2, lengths, pe, drop)
        else:
            x, t = enc_layer_fwd(p, x, pk.enc_pre, B, H, T2, lengths, drop)
        enc_tape.append(t)
    if pk.conformer:    # the running statistics moved: the inference pack, which folds BatchNorm, must be rebuilt
        modules.bump_param_generation()
    mem = _norm(x, pk.enc_norm) if pk.enc_pre else x
    return mem, _EncTrace(fe=fe_saved, tape=enc_tape, pe=pe, lengths=lengths, enc_last=x, drops=e_drop, B=B, T2=T2)


def _encoder_bwd(model, pk, tr, dx, g):
    """Backward of _encoder_fwd from dx = the gradient of the memory (bf16 [B*T', d]): encoder layers in reverse, then the
    front end's backward.  Parameter gradients go into g."""
    B, T2, H = tr.B, tr.T2, model.encoder.blocks[0].n_heads
    if pk.enc_pre:
        dx = _ln_bwd(dx, tr.enc_last, pk.enc_norm, g)
    for i in reversed(range(len(pk.enc))):
        if pk.conformer:
            dx = _conformer_block_bwd(pk.enc[i], tr.tape[i], dx, g, B, H, T2, tr.lengths, tr.pe, tr.drops[i])
        else:
            dx = enc_layer_bwd(pk.enc[i], tr.tape[i], dx, pk.enc_pre, g, B, H, T2, tr.lengths, tr.drops[i])
    model.frontend.backward(dx, pk.fe, tr.fe, g)


def _ctc_head(model, pk):
    """CTCAssistor's output layer (model/ctc.py:33-46) as head_fwd / head_bwd take it: (bf16 weight, fp32 bias, ld)."""
    lin = model.assistor.output_layer
    return pk.w(lin.weight), _f(lin.bias), model.assistor.ld_logits


_CTC_HEAD = ('assistor.output_layer.weight', 'assistor.output_layer.bias')      # its gradients' names


def _loss_scale(grad_scale, w):
    """The loss-gradient scale w * grad_scale as the kernels take it: (host factor, f32 device scalar or None).  A float
    grad_scale is folded on the host, exactly as before; a device tensor is multiplied in by the kernel."""
    if torch.is_tensor(grad_scale):
        return w, grad_scale
    return w * grad_scale, None


def _dec_fwd(dec, pk, tgt_in, mem, B, K, L, T2, lengths, drops):
    """The decoder in training mode, teacher-forced on tgt_in i64 [B*K, L] (K sequences per utterance) over the memory ->
    (the output layer's input bf16 [B*K*L, d], the last layer's output, the layers' tapes)."""
    _, dtable = dec.pos_emb.scale_and_table(L, mem.device)
    y = ops.embed_posenc(tgt_in, pk.emb, dtable, B * K * L, dec.d_model, period=L)
    tape = []
    for p, drop in zip(pk.dec, drops):
        y, t = _dec_layer_fwd(p, y, mem, pk.dec_pre, B, dec.n_heads, L, T2, lengths, drop, K)
        tape.append(t)
    last = y
    if pk.dec_pre:
        y = _norm(y, pk.dec_norm)
    return y, last, tape


def _dec_bwd(dec, pk, tgt_in, dlogits, y, last, tape, mem, dmem, g, B, K, L, T2, lengths, drops):
    """Backward of _dec_fwd and the output layer from dlogits: parameter gradients into g; returns dmem plus the decoder's
    gradient of the memory."""
    dy = head_bwd(dlogits, y, pk.wout, g, pk.wout_name, 'decoder.output_layer.bias')
    if pk.dec_pre:
        dy = _ln_bwd(dy, last, pk.dec_norm, g)
    for i in reversed(range(len(pk.dec))):
        dy, dmem = _dec_layer_bwd(pk.dec[i], tape[i], dy, dmem, mem, pk.dec_pre, g, B, dec.n_heads, L, T2, lengths, drops[i], K)
    embedding_bwd(tgt_in, dy, pk.emb, math.sqrt(dec.d_model), g, 'decoder.embedding.weight')       # decoder/transformer.py:163,169
    return dmem


def _mwer_references(truth, truth_length):
    """The sequences the n-best is scored against, as eval.py compares them: truth[b, 1 : truth_length[b]] (the transcript
    between BOS and its closing <S/E>; without truth_length, up to the first <S/E>) -> (i32 [B, L], lengths i32 [B])."""
    ref = truth[:, 1:].to(torch.int32).contiguous()
    if truth_length is not None:
        return ref, (truth_length.to(ref.device).to(torch.int32) - 1).contiguous()
    return ref, (ref == 1).int().argmax(dim=1).to(torch.int32)


def _mwer_branch(model, pk, nbest, truth, truth_length, mem, tr, drop_seed, grad_scale, g, dmem, estimator='nbest'):
    """The MWER term (DESIGN.md 4.11) on the n-best (hypothesis inputs i64 [B*K, Lp] = BOS y PAD..., targets [B*K, Lp] =
    y <S/E> -1..., K), over the memory of the cross-entropy branch: the decoder teacher-forced on the K hypotheses of each
    utterance, their token log-probs, the edit distances to the references, and with g the backward of
    sum_b L_MWER,b / B (x grad_scale) on top of dmem.  -> (mean_b L_MWER,b, dmem).  estimator 'sample': the rows are K
    samples drawn with replacement, and only the coefficients change (otb_mwer_sample_coeff: L_MWER,b = mean_k W_k and the
    score-function coefficients (W_k - mean W) / K)."""
    hyp_in, hyp_tgt, K = nbest
    dec, B, T2, lengths = model.decoder, tr.B, tr.T2, tr.lengths
    Lp = hyp_in.shape[1]
    if tuple(hyp_in.shape) != (B * K, Lp) or tuple(hyp_tgt.shape) != (B * K, Lp):
        raise ValueError(f'forward_backward: the n-best rows must be [B*K, Lp] = [{B * K}, Lp], got {tuple(hyp_in.shape)} and '
                         f'{tuple(hyp_tgt.shape)}')
    tgt = hyp_tgt.to(torch.int32).contiguous()
    n = ((tgt >= 0).sum(dim=1) - 1).to(torch.int32)                              # the length of y
    ref, ref_len = _mwer_references(truth, truth_length)
    err = ops.edit_distance(tgt, n, ref, ref_len, K)
    drops = _drops(pk.rates['decoder'], pk.attn_rates['decoder'], drop_seed, MWER_SITE, 3)
    hyp_in = hyp_in.contiguous()
    y, last, tape = _dec_fwd(dec, pk, hyp_in, mem, B, K, Lp, T2, lengths, drops)
    logits = head_fwd(y, pk.wout, pk.bout, dec.ld_logits)
    flat = tgt.view(-1)
    tok = ops.token_logprob(logits, dec.vocab_size, flat)
    ms, mdev = _loss_scale(grad_scale, 1.0 / B)
    if estimator == 'sample':
        loss_b, coeff = ops.mwer_sample_coeff(err.view(B, K), ms, mdev)
    else:
        loss_b, coeff = ops.mwer_coeff(tgt.view(B, K, Lp), n.view(B, K), err.view(B, K), tok.view(B, K, Lp), ms, mdev)
    if g is not None:
        dlogits = ops.mwer_grad(logits, dec.vocab_size, flat, tok, coeff)
        del logits
        dmem = _dec_bwd(dec, pk, hyp_in, dlogits, y, last, tape, mem, dmem, g, B, K, Lp, T2, lengths, drops)
    return loss_b.mean(), dmem


def forward_backward(model, inputs, mask, truth, truth_length=None, want_grads=True, grad_sink=None, grad_scale=1.0,
                     bf16_of=None, drop_seed=None, nbest=None, mwer_ce_weight=0.01, mwer_estimator='nbest'):
    """SpeechToText.train_pass (the contract is at the top of this file).  inputs f32 [B,T,F], mask bool [B,T], truth i64
    [B,L+1] (BOS ... EOS PAD*); the gradients are named as in model.named_parameters().  truth_length: i32/i64 [B] label
    counts incl. <S/E> (targets['targets_length'], data/loader.py:94) -- required when model.ctc_weight > 0: the loss is
    then (1 - w) * attention + w * CTC (model/speech2text.py:60-62), the CTC head's gradients flow into the encoder through
    the memory, and the CTC term alone is left on model._last_ctc_loss (None without joint CTC) for SpeechToText.forward
    to report, as the reference does.

    nbest = (hypothesis inputs i64 [B*K, Lp], their targets [B*K, Lp], K), second_pass_rows' layout: minimum word error
    rate training (DESIGN.md 4.11).  The loss becomes mean_b L_MWER,b + mwer_ce_weight * (the loss above); the decoder
    also runs on the K hypotheses of each utterance over the same memory, with its own dropout sites (MWER_SITE), and both
    branches' memory gradients go into the one encoder backward.  mwer_estimator 'nbest' (the default) is the expected risk
    over the n-best; 'sample' takes the rows as K samples from the model (SpeechToTextRecognizer.sample_ids) and trains on
    the score-function estimate: L_MWER,b = mean_k W_k, whose gradient is estimated by sum_k (W_k - mean W) / K * dl_k."""
    if mwer_estimator not in ('nbest', 'sample'):
        raise ValueError(f"forward_backward: mwer_estimator must be 'nbest' or 'sample', got {mwer_estimator!r}")
    dec = model.decoder
    ctc_w = float(getattr(model, 'ctc_weight', 0.0) or 0.0)
    if ctc_w > 0.0 and truth_length is None:
        raise ValueError('forward_backward: ctc_weight > 0 needs truth_length')
    pk = TrainPack(model, bf16_of)
    dev = inputs.device
    need_drop_seed(drop_seed, pk.rates['encoder'] + pk.rates['decoder'] + _flat(pk.attn_rates['encoder'] + pk.attn_rates['decoder']))
    ce_w = 1.0
    if nbest is not None:
        ce_w = float(mwer_ce_weight)
        if want_grads and grad_sink is None:        # two decoder passes add their gradients into the same tensors
            unused = unused_parameters(model)
            grad_sink = {n: torch.zeros(p.shape, dtype=torch.float32, device=dev) for n, p in model.named_parameters()
                         if n not in unused}

    # ------------------------------------------------------------------ forward
    mem, tr = _encoder_fwd(model, pk, inputs, mask, drop_seed)
    B, T2, lengths = tr.B, tr.T2, tr.lengths

    tgt_in = truth[:, :-1].contiguous()
    tgt_out = truth[:, 1:].contiguous()
    L = tgt_in.shape[1]
    d_drop = _drops(pk.rates['decoder'], pk.attn_rates['decoder'], drop_seed, DEC_SITE, 3)
    y, dec_last, dec_tape = _dec_fwd(dec, pk, tgt_in, mem, B, 1, L, T2, lengths, d_drop)
    V = dec.vocab_size
    logits = head_fwd(y, pk.wout, pk.bout, dec.ld_logits)
    loss_ctc, dctc = None, None
    if ctc_w > 0.0:     # CTCAssistor on the encoder states (model/ctc.py:33-52)
        wc, bc, ldc = _ctc_head(model, pk)
        cs, cdev = _loss_scale(grad_scale, ctc_w * ce_w)
        loss_ctc, _, dctc = ops.ctc_loss(head_fwd(mem, wc, bc, ldc), B, T2, V, lengths, tgt_out,
                                         truth_length.to(torch.int32).to(dev).contiguous(),
                                         model.assistor.blank, want_grad=want_grads, grad_scale=cs, scale_dev=cdev)
    model._last_ctc_loss = loss_ctc
    g, dmem = None, None
    if not want_grads:
        loss, _ = ops.ls_cross_entropy(logits, tgt_out, V, model.smoothing)
        if ctc_w > 0.0:
            loss = (1.0 - ctc_w) * loss + ctc_w * loss_ctc
    else:
        loss, dlogits = ops.ls_cross_entropy_train(logits, tgt_out, V, model.smoothing)
        att_scale, att_dev = _loss_scale(grad_scale, (1.0 - ctc_w) * ce_w)
        if att_dev is not None or att_scale != 1.0:
            # loss / accum_steps (trainer.py:216), x (1 - w)
            dlogits = ops.scale_add_table(dlogits, att_scale, scale_dev=att_dev)
        if ctc_w > 0.0:
            loss = (1.0 - ctc_w) * loss + ctc_w * loss_ctc

        # -------------------------------------------------------------- backward
        g = Grads(grad_sink)
        dmem = _dec_bwd(dec, pk, tgt_in, dlogits, y, dec_last, dec_tape, mem, dmem, g, B, 1, L, T2, lengths, d_drop)
    if nbest is not None:
        del logits, dec_tape
        loss_mwer, dmem = _mwer_branch(model, pk, nbest, truth, truth_length, mem, tr, drop_seed, grad_scale, g, dmem,
                                       mwer_estimator)
        loss = loss_mwer + ce_w * loss
    if not want_grads:
        return loss, None

    dx = dmem
    if ctc_w > 0.0:     # CTC head: parameter gradients, and its gradient with respect to the memory joins the decoder's
        dx = head_bwd(dctc, mem, wc, g, *_CTC_HEAD, resid=dmem)
    _encoder_bwd(model, pk, tr, dx, g)
    return loss, g


def ctc_forward_backward(model, inputs, mask, truth, truth_length, want_grads=True, grad_sink=None, grad_scale=1.0,
                         bf16_of=None, drop_seed=None):
    """CTCModel.train_pass: CTCModel.forward (model/ctc.py:83-96) in training mode, and its backward: front end + encoder,
    the CTC head, and nn.CTCLoss(blank 0, 'mean', zero_infinity) against truth[:, 1:-1] with truth_length - 1 labels -- the
    CTC-only model drops <S/E>, joint CTC keeps it.  The loss gradient (x grad_scale) runs back through the head into the
    shared encoder backward.  Arguments as forward_backward's; truth_length is required."""
    if truth_length is None:
        raise ValueError('ctc_forward_backward: a CTCModel needs truth_length')
    pk = EncoderPack(model, bf16_of)
    need_drop_seed(drop_seed, pk.rates['encoder'] + _flat(pk.attn_rates['encoder']))
    mem, tr = _encoder_fwd(model, pk, inputs, mask, drop_seed)
    V = model.vocab_size
    wc, bc, ld = _ctc_head(model, pk)
    tlen = (truth_length.to(inputs.device).to(torch.int32) - 1).contiguous()
    cs, cdev = _loss_scale(grad_scale, 1.0)
    loss, _, dctc = ops.ctc_loss(head_fwd(mem, wc, bc, ld), tr.B, tr.T2, V, tr.lengths, truth[:, 1:-1].contiguous(), tlen,
                                 model.assistor.blank, want_grad=want_grads, grad_scale=cs, scale_dev=cdev)
    if not want_grads:
        return loss, None
    g = Grads(grad_sink)
    _encoder_bwd(model, pk, tr, head_bwd(dctc, mem, wc, g, *_CTC_HEAD), g)
    return loss, g


# dropout site of the output of the transducer's prediction-network LSTM layer k: RNNT_SITE + k, clear of the speech
# model's (ENC_SITE, DEC_SITE, MWER_SITE and ATTN_SITE + those) and the language models' (lm.py)
RNNT_SITE = 10000
# bytes of fp32 logits the transducer's output layer holds at once: the lattice rows run through it in chunks of this size
RNNT_WORKSPACE_BYTES = 512 << 20


def lstm_layers(rnn, w, prefix):
    """The operands of an _LSTMParams stack (lm.py) named `prefix` + its parameter names: per layer the input projection
    as a Lin (bf16 W_ih, its transpose, the fp32 sum of both biases), W_hh bf16 (w casts a parameter) and the names of
    W_hh and b_hh."""
    layers = []
    for k in range(rnn.num_layers):
        w_ih = w(getattr(rnn, f'weight_ih_l{k}'))
        bias = (getattr(rnn, f'bias_ih_l{k}') + getattr(rnn, f'bias_hh_l{k}')).detach().float().contiguous()
        layers.append({'ih': Lin(w_ih, w_ih.t().contiguous(), bias, f'{prefix}weight_ih_l{k}', f'{prefix}bias_ih_l{k}'),
                       'w_hh': w(getattr(rnn, f'weight_hh_l{k}')), 'whh': f'{prefix}weight_hh_l{k}', 'bhh': f'{prefix}bias_hh_l{k}'})
    return layers


def lstm_stack_fwd(x, layers, L, N, dropout=0.0, drop_seed=None, site0=0, hidden=None, record=False, barrier=None):
    """An LSTM stack over x bf16 [L*N, I] (time-major) -> (output of the top layer bf16 [L*N, H], h_n, c_n f32 [layers, N,
    H], tape).  hidden: (h0, c0) f32 [layers, N, H] or None; with drop_seed, dropout on the output of every layer but the
    last (site site0 + k); record: keep what lstm_stack_bwd reads (per layer: input, gates, c_t, output); barrier: see
    ops.lstm_fwd.  The recurrent LM and the transducer's prediction network."""
    hs, cs, tape = [], [], []
    for k, p in enumerate(layers):
        gx = ops.linear(x, p['ih'].w, p['ih'].b, out_f32=True)
        h0 = hidden[0][k].float().contiguous() if hidden is not None else None
        c0 = hidden[1][k].float().contiguous() if hidden is not None else None
        y, h_n, c_n, gates, c_all = ops.lstm_fwd(gx, p['w_hh'], L, N, h0, c0, train=record, barrier=barrier)
        hs.append(h_n)
        cs.append(c_n)
        if record:
            tape.append((x, gates, c_all, y))
        x = y
        if drop_seed is not None and dropout > 0.0 and k + 1 < len(layers):
            x = ops.dropout_add(y, None, dropout, drop_seed, site0 + k)
    return x, torch.stack(hs), torch.stack(cs), tape


def lstm_stack_bwd(dy, tape, layers, L, N, g, dropout=0.0, drop_seed=None, site0=0):
    """Backward through time of lstm_stack_fwd(record=True, zero initial state) from dy bf16 [L*N, H]: the parameter
    gradients into g (added into its sink when it has one) -> the gradient of the stack's input bf16 [L*N, I]."""
    acc = g.sink is not None
    for k in reversed(range(len(layers))):
        p = layers[k]
        xk, gates, c_all, y = tape[k]
        dg = ops.lstm_bwd(dy, p['w_hh'], gates, c_all, L, N)
        # W_hh sees h_{t-1}: the rows of step t >= 1 against the output of step t - 1 (zero initial state)
        if L > 1:
            g[p['whh']] = ops.linear_wgrad(dg[N:], y[:-N], out=g.out(p['whh']), accumulate=acc)
        else:
            _acc_out(g, p['whh'], p['w_hh'].shape, dg.device)
        dy = linear_bwd(dg, xk, p['ih'], g)
        # both biases enter the gates alike
        if acc:
            g[p['bhh']] = ops.colsum(dg, out=g.out(p['bhh']), accumulate=True)
        else:
            g[p['bhh']] = g[p['ih'].bname].clone()
        if k > 0 and drop_seed is not None and dropout > 0.0:
            dy = ops.dropout_add(dy, None, dropout, drop_seed, site0 + k - 1)
    return dy


def transducer_operands(model, pk, simple=True):
    """The prediction network's and the joint network's operands of a TransducerModel, cast by the LayerPack pk; with
    simple and a prune_range, also the simple joint's (simple_operands) under 'simple'."""
    j, d = model.joint, model.decoder
    op = {'enc': pk._lin(j.enc_proj), 'dec_w': pk.w(j.dec_proj.weight), 'out_w': pk.w(j.output_layer.weight),
          'out_b': _f(j.output_layer.bias), 'emb': pk.w(d.embedding.weight), 'layers': lstm_layers(d.rnn, pk.w, 'decoder.rnn.')}
    if simple and j.prune_range is not None:
        op['simple'] = simple_operands(model, pk)
    return op


def simple_operands(model, pk):
    """simple_am_proj and simple_lm_proj of a pruned TransducerModel as Lin, W^T zero-padded to [K, ld_logits] so that the
    dgrad GEMM takes the padded bf16 gradient rows as they are."""
    j = model.joint
    ld, V = j.ld_logits, j.vocab_size

    def lin(m):
        x = pk._lin(m)
        wt = torch.zeros(x.w.shape[1], ld, dtype=BF16, device=x.w.device)
        wt[:, :V] = x.wt
        return x._replace(wt=wt)

    return {'am': lin(j.simple_am_proj), 'lm': lin(j.simple_lm_proj)}


def _padded_linear_bwd(dz, x, lin, V, g, resid=None):
    """linear_bwd for a Linear(K -> V) whose output gradient dz bf16 [M, ld] is zero-padded past V (lin.wt [K, ld])."""
    acc = g.sink is not None
    g[lin.wname] = ops.linear_wgrad(dz[:, :V], x, out=g.out(lin.wname), accumulate=acc)
    db = torch.zeros(dz.shape[1], dtype=torch.float32, device=dz.device)
    ops.colsum(dz, out=db, accumulate=True)
    g.put(lin.bname, db[:V])
    if resid is not None:
        return ops.linear(dz, lin.wt, None, EPI_RESID, resid=resid)
    return ops.linear(dz, lin.wt)


def _simple_joint(model, op, mem, gb, B, T2, U1, lengths, u_len, labels):
    """The pruned loss's simple joint: am = simple_am_proj(memory), lm = simple_lm_proj(g) in f32, its node log-probs,
    loss (unit gradient scale) and node gradients, and the bands s_begin i32 [B, T'] (DESIGN.md 4.22)."""
    V, ld, S = model.vocab_size, model.joint.ld_logits, model.joint.prune_range
    sp = op['simple']
    am = ops.linear(mem, sp['am'].w, sp['am'].b, EPI_BIAS, out=torch.empty(B * T2, ld, dtype=torch.float32, device=mem.device))
    lm = ops.linear(gb, sp['lm'].w, sp['lm'].b, EPI_BIAS, out=torch.empty(B * U1, ld, dtype=torch.float32, device=mem.device))
    lp, m_am, m_lm = ops.rnnt_simple_lse(am, lm, V, B, T2, U1, lengths, u_len, labels)
    loss, _, grad = ops.rnnt_loss(lp, B, T2, U1, lengths, u_len)
    s_begin = ops.rnnt_prune_ranges(grad, B, T2, U1, lengths, u_len, S)
    return loss, s_begin, (am, lm, lp, m_am, m_lm, grad)


def transducer_head(model, op, mem, B, T2, lengths, truth, truth_length, drop_seed=None, g=None, grad_scale=1.0,
                    workspace_bytes=None):
    """The transducer half above the encoder (DESIGN.md 4.22): enc_proj over the memory bf16 [B*T', d], the prediction
    network over [BLK, y_1 .. y_U] (y = truth[:, 1:-1], truth_length - 1 labels), dec_proj, the joint over the padded
    lattice [B, T', U + 1] and the RNN-T loss, with the output layer run over chunks of lattice rows holding at most
    workspace_bytes (RNNT_WORKSPACE_BYTES) of fp32 logits.  op: transducer_operands.  -> (loss 0-d f32 = mean_b nll_b,
    dmem bf16 [B*T', d] or None).  With g (a Grads) the backward runs: each chunk's logits are recomputed, turned into
    bf16 dlogits and sent through the dgrad and the accumulating wgrad GEMMs, then the joint, the projections and the
    prediction network run backward into g; the loss gradient is scaled by grad_scale (a float or an f32 device scalar).
    With the joint's prune_range S (op['simple'] present): the simple joint picks S label positions per frame on the device,
    the joint and the output layer run over the [B, T', S] band only, and the loss is simple_loss_scale * L_simple +
    L_pruned."""
    dev = mem.device
    V, D = model.vocab_size, model.joint.inner_size
    dec = model.decoder
    labels = truth[:, 1:-1].to(torch.int32).contiguous()
    u_len = (truth_length.to(dev).to(torch.int32) - 1).contiguous()
    U1 = labels.shape[1] + 1
    if U1 - 1 > ops.RNNT_MAX_LABELS:
        raise ValueError(f'transducer: transcripts of {U1 - 1} labels; at most {ops.RNNT_MAX_LABELS} are supported')
    dec._check_device(dev)
    tok = torch.cat((torch.zeros(B, 1, dtype=torch.long, device=dev), truth[:, 1:-1].to(dev)), dim=1).t().contiguous()  # [U1, B]
    want = g is not None
    x = ops.embedding(tok.view(-1), op['emb'])
    y, _, _, tape = lstm_stack_fwd(x, op['layers'], U1, B, dec.dropout, drop_seed, RNNT_SITE, record=want)
    H = y.shape[1]
    gb = y.view(U1, B, H).transpose(0, 1).contiguous().view(B * U1, H)                # utterance-major predictor rows
    enc = op['enc']
    ep = ops.linear(mem, enc.w, enc.b, EPI_BIAS)
    pp = ops.linear(gb, op['dec_w'])
    pruned = 'simple' in op
    S = model.joint.prune_range if pruned else None
    band = {}
    if pruned:
        loss_s, s_begin, simple = _simple_joint(model, op, mem, gb, B, T2, U1, lengths, u_len, labels)
        band = {'s_begin': s_begin, 'S': S}
    hj = ops.rnnt_joint(ep, pp, B, T2, U1, lengths, u_len, **band)
    rows, ld = B * T2 * (S if pruned else U1), model.joint.ld_logits
    chunk = max(8, (workspace_bytes or RNNT_WORKSPACE_BYTES) // (4 * ld) // 8 * 8)
    ws = torch.empty(min(chunk, rows), ld, dtype=torch.float32, device=dev)
    lp = torch.empty(rows, 3, dtype=torch.float32, device=dev)
    spans = [(r0, min(rows, r0 + chunk)) for r0 in range(0, rows, chunk)]

    def logits(r0, r1):
        return ops.linear(hj[r0:r1], op['out_w'], op['out_b'], EPI_BIAS, out=ws[:r1 - r0])

    for r0, r1 in spans:
        ops.rnnt_logprob(logits(r0, r1), r0, V, B, T2, U1, lengths, u_len, labels, lp, **band)
    s, sdev = _loss_scale(grad_scale, 1.0)
    loss, _, grad = ops.rnnt_loss(lp, B, T2, U1, lengths, u_len, s, sdev, **band)
    if pruned:
        alpha = model.joint.simple_loss_scale
        loss = alpha * loss_s + loss
    if not want:
        return loss, None

    dw = _acc_out(g, 'joint.output_layer.weight', op['out_w'].shape, dev)
    db = torch.zeros(ld, dtype=torch.float32, device=dev)
    wt = torch.zeros(D, ld, dtype=BF16, device=dev)
    wt[:, :V] = op['out_w'].t()
    dl = torch.empty(ws.shape, dtype=BF16, device=dev)
    dhj = torch.empty(rows, D, dtype=BF16, device=dev)
    for r0, r1 in spans:
        dz = ops.rnnt_dlogits(logits(r0, r1), r0, V, B, T2, U1, lengths, u_len, labels, lp, grad, out=dl[:r1 - r0], **band)
        ops.linear_wgrad(dz[:, :V], hj[r0:r1], out=dw, accumulate=True)
        ops.colsum(dz, out=db, accumulate=True)
        ops.linear(dz, wt, out=dhj[r0:r1])
    g.put('joint.output_layer.bias', db[:V])
    del ws, dl
    dep, dpp = ops.rnnt_joint_bwd(dhj, hj, B, T2, U1, lengths, u_len, **band)
    del dhj, hj
    dmem = linear_bwd(dep, mem, enc, g)
    acc = g.sink is not None
    g['joint.dec_proj.weight'] = ops.linear_wgrad(dpp, gb, out=g.out('joint.dec_proj.weight'), accumulate=acc)
    dgb = ops.linear(dpp, op['dec_w'].t().contiguous())
    if pruned:
        # the simple loss trains the simple projections and flows into the memory and the predictor; no gradient
        # flows through the bands
        am, lm, lp_s, m_am, m_lm, grad_s = simple
        s_s, sdev_s = _loss_scale(grad_scale, model.joint.simple_loss_scale)
        d_am, d_lm = ops.rnnt_simple_bwd(am, lm, V, B, T2, U1, lengths, u_len, labels, lp_s, m_am, m_lm, grad_s, s_s, sdev_s, ld)
        del am, lm
        dmem = _padded_linear_bwd(d_am, mem, op['simple']['am'], V, g, resid=dmem)
        dgb = _padded_linear_bwd(d_lm, gb, op['simple']['lm'], V, g, resid=dgb)
    dy = dgb.view(B, U1, H).transpose(0, 1).contiguous().view(U1 * B, H)
    dx = lstm_stack_bwd(dy, tape, op['layers'], U1, B, g, dec.dropout, drop_seed, RNNT_SITE)
    embedding_bwd(tok, dx, op['emb'], 1.0, g, 'decoder.embedding.weight')
    return loss, dmem


def transducer_forward_backward(model, inputs, mask, truth, truth_length, want_grads=True, grad_sink=None, grad_scale=1.0,
                                bf16_of=None, drop_seed=None):
    """TransducerModel.train_pass (the contract is at the top of this file): front end + encoder (_encoder_fwd), then
    transducer_head (enc_proj, the prediction network over [BLK, y], dec_proj, the joint and the chunked RNN-T loss) against
    truth[:, 1:-1] with truth_length - 1 labels, and the backward in reverse ending in _encoder_bwd.  Arguments as
    ctc_forward_backward's; truth_length is required."""
    if truth_length is None:
        raise ValueError('transducer_forward_backward: a TransducerModel needs truth_length')
    pk = EncoderPack(model, bf16_of, with_decoder=False)
    need_drop_seed(drop_seed, pk.rates['encoder'] + _flat(pk.attn_rates['encoder']) + [model.decoder.dropout])
    op = transducer_operands(model, pk)
    mem, tr = _encoder_fwd(model, pk, inputs, mask, drop_seed)
    g = Grads(grad_sink) if want_grads else None
    loss, dmem = transducer_head(model, op, mem, tr.B, tr.T2, tr.lengths, truth, truth_length, drop_seed, g, grad_scale)
    if not want_grads:
        return loss, None
    _encoder_bwd(model, pk, tr, dmem, g)
    return loss, g


def mixspeech_halves(model, inputs, mask, truth, truth_length=None, *, seed, step, scale, lam):
    """mix_batch of the speech models (SpeechToText, CTCModel): MixSpeech (trainer.py:155-201) on a batch as train_batch
    returns it.  With P = B // 2 pairs (an odd last utterance is dropped) and lambda ~ Beta(1/2, 1/2) drawn on the device
    from the i32 device scalars seed / step, otb_mixspeech makes x_mix = lambda x[0::2] + (1 - lambda) x[1::2] and mask_mix
    = mask[0::2] | mask[1::2]; lam (f32 [3]) receives {lambda, lambda * scale, (1 - lambda) * scale}.  -> the batches of
    the two passes, (x_mix, mask_mix, truth[0::2], truth_length[0::2]) and the same with [1::2]: pass 1 is weighted by
    lambda and pass 2 by 1 - lambda (their loss-gradient scales are lam[1] and lam[2]).  B < 2 raises ValueError."""
    if inputs.dim() != 3:
        raise ValueError(f'MixSpeech mixes [B, T, F] features, got inputs of shape {tuple(inputs.shape)}')
    B = inputs.shape[0]
    if B < 2:
        raise ValueError('MixSpeech mixes pairs of utterances: it needs a batch of at least 2')
    n = B // 2 * 2
    x_mix, m_mix = ops.mixspeech(inputs.contiguous().float(), mask.contiguous(), seed, step, scale, lam)

    def half(k):
        tl = None if truth_length is None else truth_length[k:n:2].contiguous()
        return x_mix, m_mix, truth[k:n:2].contiguous(), tl

    return half(0), half(1)


def next_drop_seed(model, device):
    """The dropout seed of the next training forward (a fresh mask per forward), on the device."""
    seed = getattr(model, '_drop_seed', None)
    if seed is None or seed.device != device:
        seed = torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32).to(device)
        model._drop_seed = seed
    seed.add_(1)
    return seed


class _TrainingLoss(torch.autograd.Function):
    """loss = model.train_pass(*batch) as ONE autograd node over the fp32 master parameters."""

    @staticmethod
    def forward(ctx, model, batch, names, *params):
        with torch.no_grad():
            loss, grads = model.train_pass(*batch, drop_seed=next_drop_seed(model, batch[0].device))
        ctx.grads = [grads.get(n) for n in names]
        ctx.shapes = [p.shape for p in params]
        return loss.clone()

    @staticmethod
    def backward(ctx, gloss):
        return (None, None, None) + tuple(None if gr is None else gr.view(shp) * gloss
                                          for gr, shp in zip(ctx.grads, ctx.shapes))


def loss_with_grad(model, *batch):
    """A model's forward in training mode with gradients enabled: the loss tensor whose .backward() fills `.grad` of every
    parameter."""
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    return _TrainingLoss.apply(model, batch, [n for n, _ in named], *[p for _, p in named])


def loss_train_mode(model, *batch):
    """A model's forward in training mode without gradients (model.train() under torch.no_grad(), e.g. a validation loop
    that does not call eval()): the forward the reference runs in train() -- dropout on, a Conformer's BatchNorm with the
    batch statistics and its running statistics updated -- with no backward.  -> loss."""
    with torch.no_grad():
        return model.train_pass(*batch, want_grads=False, drop_seed=next_drop_seed(model, batch[0].device))[0]


def _check_mwer(model, nbest, ce_weight, max_len, mixspeech, name='mwer_nbest'):
    """What FusedTrainer refuses for minimum word error rate training, before any device work (name: the option that sets
    K, mwer_nbest or mwer_samples)."""
    if not isinstance(getattr(model, 'decoder', None), TransformerDecoder):
        raise NotImplementedError(f'MWER training scores an attention decoder\'s n-best; {type(model).__name__} has none')
    if not 2 <= nbest <= 16:
        raise ValueError(f'{name} must be 0 (off) or in 2..16, got {nbest}')
    if not ce_weight >= 0.0:
        raise ValueError(f'mwer_ce_weight must be >= 0, got {ce_weight}')
    if not 1 <= max_len <= 1022:
        raise ValueError(f'mwer_max_len must be in 1..1022, got {max_len}')
    if mixspeech:
        raise NotImplementedError('MWER training and MixSpeech are two different pairs of passes; choose one')


def transformer_lr(step, model_size, warmup_steps, factor=1.0):
    """TransformerScheduler.get_step_lr (otrans/train/scheduler.py:137-138)."""
    return factor * model_size ** (-0.5) * min(step ** (-0.5), step * warmup_steps ** (-1.5))


class FusedTrainer:
    """The inner step of Trainer.train_one_epoch (trainer.py:206-234) on flat fp32 buffers:
    forward + hand-written backward -> (data-parallel) gradient all-reduce over NCCL -> global-norm clip + Adam in two
    kernels, no host synchronisation.  Parameters become views into one flat buffer (state_dict keys / shapes unchanged).
    `model` is any model with the training contract at the top of this file.

    mixspeech=True (run.py -ms, trainer.py:155-201): every micro-step mixes pairs of utterances with lambda ~ Beta(1/2,
    1/2) drawn on the device (model.mix_batch) and runs the model twice on the mix, once per target half, each pass with
    its own dropout seed; the loss is lambda L1 + (1 - lambda) L2.  Speech models only (NotImplementedError otherwise).
    `last_lambda` is the device scalar of the last micro-step's lambda.
    grad_noise = sigma > 0 (train: grad_noise, trainer.py:223-227): sigma / accum_steps * N(0, 1) is added to every trained
    gradient element after the clip and before Adam, inside the fused Adam launch.  The reference's loop adds it to every
    parameter with requires_grad and raises TypeError on a Conformer, whose post_ffn parameters have no gradient; this
    trainer leaves them out (unused_parameters) and adds noise to what it trains.
    mwer_nbest = K in 2..16: minimum word error rate training (DESIGN.md 4.11).  Every micro-step first decodes the
    micro-batch's K-best with the current weights (beam_width = nbest = K, penalty 0, max_len = mwer_max_len) on the
    inference path, in eval mode and outside any CUDA graph, then trains on mean_b L_MWER,b + mwer_ce_weight * (the
    model's loss).  Attention-decoder models only (NotImplementedError otherwise); not with mixspeech.
    mwer_samples = K in 2..16: sampling-based MWER training (DESIGN.md 4.11), in place of mwer_nbest (not with it).  Every
    micro-step draws K samples per utterance from the model (SpeechToTextRecognizer.sample_ids, eval mode, outside any
    CUDA graph, max_len = mwer_max_len) and trains on mean_b mean_k W_k + mwer_ce_weight * (the model's loss) through the
    score-function gradient.  The sampling seed is an i32 device scalar advanced every micro-step, the same on every rank;
    each rank draws with it XOR a constant of its own, so the ranks' samples are independent.  state_dict saves it
    ('sample_seed'), so a resumed run draws the same samples on every rank."""

    def __init__(self, model, lr=1e-3, betas=(0.9, 0.98), eps=1e-9, weight_decay=1e-6, clip_grad=5.0, model_size=256,
                 warmup_steps=12000, factor=1.0, accum_steps=1, process_group=None, use_graph=True, mixspeech=False,
                 grad_noise=0.0, mwer_nbest=0, mwer_ce_weight=0.01, mwer_max_len=60, mwer_samples=0):
        if mixspeech and not hasattr(model, 'mix_batch'):
            raise NotImplementedError(f'MixSpeech mixes [B, T, F] speech features; {type(model).__name__} takes token inputs')
        if not grad_noise >= 0.0:
            raise ValueError(f'grad_noise must be >= 0, got {grad_noise}')
        if mwer_nbest and mwer_samples:
            raise ValueError('mwer_nbest and mwer_samples are the two MWER estimators (n-best and sampled); choose one')
        if mwer_nbest:
            _check_mwer(model, mwer_nbest, mwer_ce_weight, mwer_max_len, mixspeech)
        if mwer_samples:
            _check_mwer(model, mwer_samples, mwer_ce_weight, mwer_max_len, mixspeech, name='mwer_samples')
        model.check_fused_trainer()
        self.model = model
        # parameters the forward never reads (a Conformer's post_ffn) stay out of the flat buffers: no gradient, no weight decay
        unused = unused_parameters(model)
        self.params = [(n, p) for n, p in model.named_parameters() if p.requires_grad and n not in unused]
        dev = self.params[0][1].device
        # every parameter starts on a multiple of 8 elements: the kernels that write the fp32 gradient views (wgrad, colsum)
        # and read the bf16 weight views through TMA need 16-byte aligned rows, whatever the sizes before them (an odd-sized
        # bias such as the 4234-wide output bias would otherwise misalign the CTC head's weight that follows it).
        # The gaps hold zeros, which the norm and the Adam step leave at zero.
        span = {n: (p.numel() + 7) // 8 * 8 for n, p in self.params}
        total = sum(span.values())
        self.flat_p = torch.zeros(total, dtype=torch.float32, device=dev)
        self.flat_g = torch.zeros(total, dtype=torch.float32, device=dev)
        self.m = torch.zeros(total, dtype=torch.float32, device=dev)
        self.v = torch.zeros(total, dtype=torch.float32, device=dev)
        self.sumsq = torch.zeros(1, dtype=torch.float32, device=dev)
        self.flat_bf16 = torch.empty(total, dtype=BF16, device=dev)      # ONE cast of the master weights per micro-step
        self.offsets = {}
        o = 0
        with torch.no_grad():
            for n, p in self.params:
                k = p.numel()
                self.flat_p[o:o + k].copy_(p.detach().reshape(-1))
                p.data = self.flat_p[o:o + k].view_as(p)            # parameters now alias the flat buffer
                self.offsets[n] = (o, k)
                o += span[n]
        self.sink = {n: self.flat_g[o:o + k].view_as(p) for (n, p), (o, k) in zip(self.params, [self.offsets[n] for n, _ in self.params])}
        self._by_ptr = {p.data_ptr(): (self.offsets[n], p.shape) for n, p in self.params}
        self.betas, self.eps, self.wd, self.clip = betas, eps, weight_decay, clip_grad
        self.base_lr, self.model_size, self.warmup, self.factor = lr, model_size, warmup_steps, factor
        self.accum_steps = accum_steps
        self.group = process_group
        # BaseScheduler starts at global_step 1 and its constructor already calls step() once (scheduler.py:22,42-46);
        # the trainer steps it again before every optimizer.step() (trainer.py:232): the first update uses lr(3)
        # The counts live on the DEVICE ({optimizer steps, scheduler global_step, skipped}): the fused Adam launch advances them
        # only when the gradient norm is finite, as the reference skips scheduler.step() together with optimizer.step()
        # (trainer.py:229-233) -- no host sync, and a skipped step cannot desynchronise the LR schedule / bias correction.
        self.counters = torch.tensor([0, 2, 0], dtype=torch.int32, device=dev)
        self.hyper = torch.zeros(4, dtype=torch.float32, device=dev)
        self.micro = 0
        # dropout seed of the current micro-step, on the device: incremented inside the (captured) micro-step, so every
        # CUDA-graph replay draws fresh masks (a seed passed by value would be frozen into the graph)
        self.drop_seed = torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32).to(dev)
        self.use_graph = use_graph
        self.graph_after = 2          # capture a CUDA graph for an input geometry once it has been seen this many times
        self.max_graphs = 8           # LRU bound: every graph owns a private pool with the whole activation tape
        self._graphs = {}             # key -> (graphs.CapturedStep of _micro, its static batch), most recently used last
        self._seen = {}
        # training-mode BatchNorm buffers (Conformer): updated by every micro-step, inside the graph when one is replayed
        self.bn_buffers = [t for n, t in model.named_buffers() if n.startswith('encoder.') and
                           n.rsplit('.', 1)[-1] in ('running_mean', 'running_var', 'num_batches_tracked')]
        # MixSpeech: lambda is a counter hash of (mix seed, micro-step), both on the device; last_lambda holds {lambda,
        # lambda / accum_steps, (1 - lambda) / accum_steps}, the last two the loss-gradient scales of the two passes
        self.mixspeech = bool(mixspeech)
        self.grad_noise = float(grad_noise)
        self.mix_seed = self.mix_step = self._lam = self.noise_seed = self.noise_mask = None
        if self.mixspeech:
            self.mix_seed = torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32).to(dev)
            self.mix_step = torch.zeros(1, dtype=torch.int32, device=dev)
            self._lam = torch.zeros(3, dtype=torch.float32, device=dev)
        if self.grad_noise > 0.0:
            # every rank must add the same noise (the reference seeds all ranks alike, run.py:23-26)
            self.noise_seed = torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32).to(dev)
            self.noise_mask = ops.noise_bitmask(total, [self.offsets[n] for n, _ in self.params]).to(dev)
        broadcast_from_first_([t for t in (self.mix_seed, self.noise_seed) if t is not None], process_group)
        self.mwer_nbest, self.mwer_ce_weight = int(mwer_nbest), float(mwer_ce_weight)
        self.mwer_samples = int(mwer_samples)
        self._recognizer = self.sample_seed = None
        if self.mwer_samples:
            # one base seed on every rank, so that the one value state_dict saves resumes every rank; each rank draws with
            # base ^ (rank * 0x9E3779B9), because the sampling hash keys on row ids that are local to a rank and the ranks'
            # samples must be independent (rank 0 draws with the base itself)
            self.sample_seed = torch.randint(0, 2 ** 31 - 1, (1,), dtype=torch.int32).to(dev)
            broadcast_from_first_([self.sample_seed], process_group)
            off = (rank_in(process_group) * 0x9E3779B9) & 0xFFFFFFFF
            self._seed_xor = off - 2 ** 32 if off >= 2 ** 31 else off
        if self.mwer_nbest or self.mwer_samples:
            from .recognize import SpeechToTextRecognizer
            training = model.training
            # one cached BeamDecoder: ragged batches bring a new frame count almost every step, and a decoder kept for an
            # older one would hold its KV caches and the bf16 weights of the step it last decoded; the weights move every
            # optimizer step, so a kept decoder would only save its buffer allocation
            K = self.mwer_nbest or self.mwer_samples
            self._recognizer = SpeechToTextRecognizer(model, beam_width=K, nbest=K, max_len=mwer_max_len, penalty=0, ngpu=0,
                                                      max_decoders=1)
            model.train(training)

    @property
    def opt_steps(self):
        return int(self.counters[0].item())

    @property
    def global_step(self):
        return int(self.counters[1].item())

    @property
    def skipped_steps(self):
        return int(self.counters[2].item())

    def lr(self):
        if self.warmup:
            return transformer_lr(self.global_step, self.model_size, self.warmup, self.factor)
        return self.base_lr

    @property
    def last_lambda(self):
        """MixSpeech's lambda of the last micro-step: f32 0-d device tensor (None without mixspeech)."""
        return None if self._lam is None else self._lam[0]

    def _bf16_of(self, param):
        (o, k), shape = self._by_ptr[param.data_ptr()]
        return self.flat_bf16[o:o + k].view(shape)

    def _micro(self, batch):
        """forward + backward of one micro-batch (what model.train_batch returned); gradients / accum_steps are ADDED into
        the flat buffer by the backward kernels themselves (no per-parameter add)."""
        self.flat_bf16.copy_(self.flat_p)
        if self.mixspeech:
            return self._micro_mix(batch)
        self.drop_seed.add_(1)
        kw = {}
        if self.mwer_nbest:         # the n-best rows ride at the end of the batch (_with_nbest)
            batch, kw = batch[:-2], {'nbest': batch[-2:] + (self.mwer_nbest,), 'mwer_ce_weight': self.mwer_ce_weight}
        elif self.mwer_samples:     # so do the sampled rows
            batch, kw = batch[:-2], {'nbest': batch[-2:] + (self.mwer_samples,), 'mwer_ce_weight': self.mwer_ce_weight,
                                     'mwer_estimator': 'sample'}
        loss, _ = self.model.train_pass(*batch, grad_sink=self.sink, grad_scale=1.0 / self.accum_steps, bf16_of=self._bf16_of,
                                        drop_seed=self.drop_seed, **kw)
        return loss

    def _with_nbest(self, batch):
        """MWER: the micro-batch's K-best (mwer_samples: K samples) decoded with the current weights on the inference path
        (eval mode, so no dropout and a Conformer's BatchNorm on its running statistics), appended to the batch as second_pass_rows' rows
        (hypothesis inputs i64 [B*K, Lp], targets i32 [B*K, Lp]).  Reading Lp is a host synchronisation; as part of the
        batch the rows make Lp and K part of the CUDA-graph key."""
        from .recognize import second_pass_rows
        enc = self.model.encoder
        maps, enc.return_attn_weights = enc.return_attn_weights, False    # training produces no attention maps
        self.model.eval()
        try:
            if self.mwer_samples:
                self.sample_seed.add_(1)            # fresh samples every micro-step, without a host synchronisation
                seed = self.sample_seed if not self._seed_xor else torch.bitwise_xor(self.sample_seed, self._seed_xor)
                ids, _, _ = self._recognizer.sample_ids(batch[0], batch[1], self.mwer_samples, seed)
            else:
                ids, _, _ = self._recognizer.recognize_ids(batch[0], batch[1])
        finally:
            self.model.train()
            enc.return_attn_weights = maps
        hyp_in, tgt, _, Lp = second_pass_rows(ids)
        return batch + (hyp_in, tgt.view(-1, Lp))

    def _micro_mix(self, batch):
        """MixSpeech micro-step: the mix, then two passes over it (not one merged 2P-row pass: the reference's two forwards
        draw independent dropout masks and update a Conformer's BatchNorm statistics twice), their gradients scaled by
        lambda / accum_steps and (1 - lambda) / accum_steps on the device.  lambda never goes to the host."""
        self.mix_step.add_(1)
        halves = self.model.mix_batch(*batch, seed=self.mix_seed, step=self.mix_step, scale=1.0 / self.accum_steps, lam=self._lam)
        losses = []
        for k, half in enumerate(halves):
            self.drop_seed.add_(1)
            loss, _ = self.model.train_pass(*half, grad_sink=self.sink, grad_scale=self._lam[1 + k], bf16_of=self._bf16_of,
                                            drop_seed=self.drop_seed)
            losses.append(loss)
        lam = self._lam[0]
        return lam * losses[0] + (1 - lam) * losses[1]         # trainer.py:197

    def _graph_for(self, batch):
        """The ~870 launches of one micro-batch captured once per input geometry and replayed: launched one by one from
        Python the step is host-bound.
        Real ASR batches have a new (T, L) almost every step, so a geometry runs EAGERLY until its `graph_after`-th
        sighting, which runs eagerly on the static inputs and captures (graphs.CapturedStep): replays start at the next
        sighting.  At most `max_graphs` graphs are kept (least recently used first out): use_graph pays off with bucketed /
        padded batches (otrans/data/bucket.py), it must not grow memory without bound otherwise.
        Returns None when this call should run eagerly, else (the captured micro-step, its static inputs)."""
        dev = batch[0].device
        key = tuple(None if t is None else tuple(t.shape) for t in batch) + (dev.index,)
        if key not in self._graphs:
            n = self._seen.get(key, 0) + 1
            if len(self._seen) > 4096:
                self._seen.clear()
            self._seen[key] = n
            if n < self.graph_after:
                return None

        return lru_get(self._graphs, key, self.max_graphs,         # evicting a graph drops its memory pool
                       lambda: (CapturedStep(self._micro), tuple(None if t is None else t.to(dev).clone() for t in batch)))

    # ---- optimizer state: the reference's checkpoint (trainer.py:280-290, loaded by run.py:54-61 with -ct -ios) ----

    def _torch_adam(self):
        """A torch.optim.Adam over the reference's parameter list (run.py:42-44: every parameter with requires_grad, a
        Conformer's post_ffn included) with this trainer's hyper-parameters and no state."""
        params = [p for p in self.model.parameters() if p.requires_grad]
        return torch.optim.Adam(params, lr=self.lr(), betas=self.betas, eps=self.eps, weight_decay=self.wd)

    def state_dict(self):
        """{'global_step', 'optim', 'fused_trainer'} -- what the reference's save_optimizer_state_dict writes, plus this
        trainer's own counters.  'optim' is torch.optim.Adam.state_dict() of the reference's parameter list, built by torch
        itself from the flat buffers (exp_avg, exp_avg_sq and step of every trained parameter; a parameter the trainer
        leaves out, such as a Conformer's post_ffn, keeps its index and has no state, as torch's Adam leaves a parameter
        whose gradient stays None), so run.py -ct -ios loads the file unchanged.  'fused_trainer' holds the skipped steps
        and the random state (dropout seed, MixSpeech seed and micro-step, noise seed), so that a resumed run continues the
        same sequence.  Save at the end of an accumulation window: a gradient still accumulating is not saved (the
        reference does not save it either)."""
        t, global_step, skipped = self.counters.tolist()
        opt = self._torch_adam()
        by_id = {id(p): n for n, p in self.model.named_parameters()}
        if t > 0:
            for p in opt.param_groups[0]['params']:
                n = by_id[id(p)]
                if n not in self.offsets:
                    continue
                o, k = self.offsets[n]
                opt.state[p] = {'step': torch.tensor(float(t)), 'exp_avg': self.m[o:o + k].view(p.shape).clone(),
                                'exp_avg_sq': self.v[o:o + k].view(p.shape).clone()}

        def host(x):
            return None if x is None else int(x.reshape(-1)[0])

        own = {'skipped_steps': skipped, 'drop_seed': host(self.drop_seed), 'mix_seed': host(self.mix_seed),
               'mix_step': host(self.mix_step), 'noise_seed': host(self.noise_seed)}
        if self.sample_seed is not None:
            own['sample_seed'] = host(self.sample_seed)
        return {'global_step': global_step, 'optim': opt.state_dict(), 'fused_trainer': own}

    def load_state_dict(self, ckpt):
        """Resume from state_dict()'s format, or a file the reference's Trainer wrote ({'global_step', 'optim'}): Adam's
        moments go into the flat buffers and counters = [Adam step, global_step, skipped or 0], so the next update uses
        lr(global_step + 1) and Adam step + 1, as the reference's does after run.py -ct -ios.  The file's betas, eps and
        weight_decay replace the constructor's, as torch's loader does; the learning rate stays this trainer's schedule.
        The file is validated by torch.optim.Adam.load_state_dict after these refusals (ValueError, before any device work):
        no 'global_step', a different parameter count or shape, amsgrad, unequal step counts over the trained parameters."""
        if 'global_step' not in ckpt:
            raise ValueError("optimizer checkpoint without 'global_step' (trainer.py:280-288 writes it)")
        sd = ckpt['optim']
        groups = sd['param_groups']
        named = [(n, p) for n, p in self.model.named_parameters() if p.requires_grad]
        ids = [i for g in groups for i in g['params']]
        if len(ids) != len(named):
            raise ValueError(f'optimizer checkpoint for {len(ids)} parameters, this model trains {len(named)}')
        if any(g.get('amsgrad', False) for g in groups):
            raise ValueError('optimizer checkpoint with amsgrad=True: FusedTrainer runs plain Adam')
        steps = set()
        for pid, (n, p) in zip(ids, named):
            st = sd['state'].get(pid)
            if st is None:
                if n in self.offsets:
                    steps.add(0)
                continue
            for key in ('exp_avg', 'exp_avg_sq'):
                if tuple(st[key].shape) != tuple(p.shape):
                    raise ValueError(f'optimizer checkpoint: {key} of {n} has shape {tuple(st[key].shape)}, the parameter '
                                     f'{tuple(p.shape)}')
            if n in self.offsets:
                steps.add(int(float(st['step'])))
        if len(steps) > 1:
            raise ValueError(f'optimizer checkpoint with unequal Adam step counts over the trained parameters: {sorted(steps)}')
        opt = self._torch_adam()
        opt.load_state_dict(sd)
        g = opt.param_groups[0]
        self.betas, self.eps, self.wd = tuple(g['betas']), g['eps'], g['weight_decay']
        t = steps.pop() if steps else 0
        with torch.no_grad():
            self.m.zero_()
            self.v.zero_()
            for n, p in named:
                st = opt.state.get(p)
                if n not in self.offsets or not st:
                    continue
                o, k = self.offsets[n]
                self.m[o:o + k].copy_(st['exp_avg'].reshape(-1))
                self.v[o:o + k].copy_(st['exp_avg_sq'].reshape(-1))
            own = ckpt.get('fused_trainer') or {}
            self.counters.copy_(torch.tensor([t, int(ckpt['global_step']), int(own.get('skipped_steps', 0))], dtype=torch.int32))
            for name in ('drop_seed', 'mix_seed', 'mix_step', 'noise_seed', 'sample_seed'):
                dst = getattr(self, name)
                if dst is not None and own.get(name) is not None:
                    dst.fill_(int(own[name]))
            self.flat_g.zero_()
        self.micro = 0

    def step(self, *batch, truth_length=None):
        """One micro-batch; every `accum_steps` calls an optimizer step.  Returns the (un-scaled) loss tensor.
        The arguments are the model's batch, which its train_batch validates (TypeError): step(inputs, mask, truth,
        truth_length=None) for a SpeechToText, truth_length (targets['targets_length']) needed by joint-CTC models only;
        the same with truth_length required for a CTCModel; step(inputs, targets), i64 [N, L] each (the reference's
        inputs['inputs'] and targets['targets']), for a TransformerLanguageModel."""
        if truth_length is not None:
            batch += (truth_length,)
        batch = self.model.train_batch(*batch)
        if self.mixspeech and batch[0].shape[0] < 2:
            raise ValueError('MixSpeech mixes pairs of utterances: it needs a batch of at least 2')
        with torch.no_grad():
            # data parallel: BatchNorm running statistics follow the first rank's (DistributedDataParallel's
            # broadcast_buffers): each rank's forward updates them from its own shard, so they would drift apart
            broadcast_from_first_(self.bn_buffers, self.group)
            if self.mwer_nbest or self.mwer_samples:
                batch = self._with_nbest(batch)
            ent = self._graph_for(batch) if self.use_graph else None
            if ent is not None:
                micro, static = ent
                for s, t in zip(static, batch):
                    if s is not None:
                        s.copy_(t)
                loss = micro(static)
                if self.bn_buffers:
                    modules.bump_param_generation()     # a replay moved the running statistics
            else:
                loss = self._micro(batch)
            self.micro += 1
            if self.micro % self.accum_steps == 0:
                # the one exchange step of data-parallel training (SURVEY.md 8e): mean of the flat gradient over ranks,
                # ONE NCCL all-reduce per optimizer step (the reference's DDP reduces on every micro-batch)
                allreduce_mean_(self.flat_g, self.group)
                ops.sumsq(self.flat_g, self.sumsq)
                ops.adam_step_sched(self.flat_p, self.flat_g, self.m, self.v, self.sumsq, self.clip, self.base_lr, self.model_size,
                                    self.warmup, self.factor, self.betas, self.eps, self.wd, self.counters, self.hyper,
                                    noise_std=self.grad_noise / self.accum_steps, noise_seed=self.noise_seed,
                                    noise_mask=self.noise_mask)
                self.flat_g.zero_()
                modules.bump_param_generation()     # bf16 shadow copies (modules._Packed) must be rebuilt
        return loss
