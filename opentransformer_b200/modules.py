"""Host-side mirror of the reference's nn.Module surface for the hot path.

Same class names, constructor kwargs (the YAML sub-dicts verbatim) and ``state_dict()`` key names /
shapes as the reference so existing checkpoints load unchanged (SURVEY.md 8b):

    ConvFrontEnd        <- otrans/frontend/conv.py:86-159
    ConcatFeatureFrontEnd, ConcatWithLinearFrontEnd <- otrans/frontend/concat.py:11-56
    TransformerEncoder  <- otrans/encoder/transformer.py:93-134
    TransformerDecoder  <- otrans/decoder/transformer.py:129-208

The nn.Linear / nn.LayerNorm / nn.Conv2d / nn.Embedding objects below are *parameter holders*
only (they give identical key names and default init); their ``forward`` is never called.  All
compute goes through ``ops`` -> libotb200.so (hand-written sm_90a kernels).  There is no CPU path:
calling a module with CPU tensors raises.

Numerics: GEMM operands / activations are bf16, accumulation fp32, LayerNorm / softmax statistics
fp32 (DESIGN.md "rounding points").  The module-level forward is the inference path; training goes through
``SpeechToText.forward`` in train mode -> train.py (hand-written backward).
"""
import math

import torch
import torch.nn as nn

from . import ops
from .ops import BF16, EPI_BIAS, EPI_GLU, EPI_RELU, EPI_RESID, EPI_RESID_LN, EPI_TABLE, ACT_EPILOGUE


def _lengths(mask):
    """bool [B,T] prefix mask -> int32 [B] lengths (masks are contiguous prefixes, SURVEY.md 8a)."""
    return mask.sum(dim=1).to(torch.int32).contiguous()


_PARAM_GENERATION = [0]


def bump_param_generation():
    """Invalidate every bf16 shadow copy: called after parameters were updated outside torch's version tracking
    (the fused Adam kernel of train.FusedTrainer writes the flat fp32 buffer directly)."""
    _PARAM_GENERATION[0] += 1


class _Packed:
    """bf16 shadow copies of fp32 master parameters, refreshed when any parameter changes
    (load_state_dict / optimizer steps bump ``Tensor._version``)."""

    def __init__(self, module, builder):
        self._module, self._builder, self._sig, self._val = module, builder, None, None

    def get(self):
        sig = (_PARAM_GENERATION[0],) + tuple((p.data_ptr(), p._version) for p in self._module.parameters())
        if self._val is None or sig != self._sig:
            with torch.no_grad():
                self._val = self._builder()
            self._sig = sig
        return self._val


def _w(lin):
    return lin.weight.detach().to(BF16).contiguous()


def _b(lin):
    return lin.bias.detach().float().contiguous() if lin.bias is not None else None


def _ln(norm):
    return norm.weight.detach().float().contiguous(), norm.bias.detach().float().contiguous()


def _no_train(module):
    if module.training and torch.is_grad_enabled():
        raise NotImplementedError('module-level forward is the inference path: call under model.eval() / torch.no_grad(); '
                                  'training runs through SpeechToText.forward (opentransformer_b200.train)')


# ------------------------------------------------------------------------------------------------
# front end
# ------------------------------------------------------------------------------------------------
CONV_KERNELS, CONV_STRIDES = range(1, 8), range(1, 5)


def _conv_pair(v):
    """An int or a [time, freq] pair, as nn.Conv2d reads kernel_size and stride."""
    return (int(v), int(v)) if isinstance(v, int) else (int(v[0]), int(v[1]))


def conv_frontend_geometry(layers, T=None, F=None):
    """The conv front end's geometry (frontend/conv.py:10-11,27,78-83), for layers = ((kt1, kf1, st1, sf1), (kt2, kf2, st2,
    sf2)).  Padding is (0, kf // 2): time is never padded.  Returns a dict:
      'geom'   the 8 ints the CUDA entry points take;
      'window' (stride, width): output frame t sees input frames [stride t, stride t + width);
      'mask'   per layer (start, step): the reference's mask[:, kt // 2 :: st][:, :t];
    and, given T and F, 'sizes' [(T1, F1), (T2, F2)] with n' = (n + 2 p - k) // s + 1 per axis.  A kernel or stride
    outside 1..7 / 1..4 raises NotImplementedError; a T too short for one output frame raises ValueError (the reference's
    conv2d raises there too)."""
    (kt1, kf1, st1, sf1), (kt2, kf2, st2, sf2) = layers
    if not all(k in CONV_KERNELS for k in (kt1, kf1, kt2, kf2)) or not all(s in CONV_STRIDES for s in (st1, sf1, st2, sf2)):
        raise NotImplementedError(f'conv front end: kernel sizes 1..7 and strides 1..4 per axis are supported, got kernels '
                                  f'({kt1}, {kf1}), ({kt2}, {kf2}) and strides ({st1}, {sf1}), ({st2}, {sf2})')
    g = {'geom': (kt1, kf1, st1, sf1, kt2, kf2, st2, sf2), 'window': (st1 * st2, kt1 + (kt2 - 1) * st1),
         'mask': ((kt1 // 2, st1), (kt2 // 2, st2))}
    if T is not None:
        sizes = []
        for kt, kf, st, sf in layers:
            if T < kt:
                raise ValueError(f'conv front end: {T} frames are too short for a {kt}-frame kernel')
            T, F = (T - kt) // st + 1, (F + 2 * (kf // 2) - kf) // sf + 1
            sizes.append((T, F))
        g['sizes'] = sizes
    return g


class Conv2dLayer(nn.Module):
    """Parameter holder with the reference's key names (frontend/conv.py:15-48).  act_func_type is accepted and ignored:
    the reference applies F.relu whatever it says (conv.py:64).  dropout is the identity at inference."""

    def __init__(self, input_size, in_channel, out_channel, kernel_size, stride, dropout=0.1, batch_norm=False,
                 residual=False, act_func_type='relu'):
        super().__init__()
        if batch_norm or residual:
            raise NotImplementedError('ConvFrontEnd never sets batch_norm / residual')
        (kt, kf), (st, sf) = _conv_pair(kernel_size), _conv_pair(stride)
        self.kernel_size, self.stride, self.dropout_p = kernel_size, stride, dropout
        self.conv_layer = nn.Conv2d(in_channel, out_channel, (kt, kf), stride=(st, sf), padding=(0, kf // 2))
        self.output_size = (input_size + 2 * (kf // 2) - kf) // sf + 1
        self.out_channel = out_channel


class ConvFrontEnd(nn.Module):
    """forward(x f32 [B,T,F], mask bool [B,T]) -> (f32 [B,T',D], bool [B,T'])   (frontend/conv.py:86-153).
    Each layer's kernel_size and stride is an int or a [time, freq] pair, kernels 1..7 and strides 1..4
    (conv_frontend_geometry)."""

    def __init__(self, input_size, output_size, in_channel=1, mid_channel=32, out_channel=128,
                 kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                 front_end_layer_norm=False):
        super().__init__()
        assert isinstance(kernel_size, list) and len(kernel_size) == 2
        assert isinstance(stride, list) and len(stride) == 2
        if in_channel != 1:
            raise NotImplementedError('in_channel must be 1 (log-fbank input)')
        self.input_size, self.output_size = input_size, output_size
        self.front_end_layer_norm = front_end_layer_norm
        self.dropout = dropout
        self.layers = tuple(_conv_pair(k) + _conv_pair(s) for k, s in zip(kernel_size, stride))
        self.geom = conv_frontend_geometry(self.layers)['geom']
        self.conv1 = Conv2dLayer(input_size, in_channel, mid_channel, kernel_size[0], stride[0], dropout)
        self.conv2 = Conv2dLayer(self.conv1.output_size, mid_channel, out_channel, kernel_size[1], stride[1], dropout)
        self.conv_output_size = self.conv2.output_size * out_channel
        self.output_layer = nn.Linear(self.conv_output_size, output_size)
        if front_end_layer_norm:
            self.layer_norm = nn.LayerNorm(output_size)
        self._pack = _Packed(self, self._build_pack)

    def _build_pack(self):
        c1 = self.conv1.conv_layer
        c2 = self.conv2.conv_layer
        C1, C2 = c1.out_channels, c2.out_channels
        F2 = self.conv2.output_size
        kt1, kf1, _, _, kt2, kf2, _, _ = self.geom
        C1p = (C1 + 63) // 64 * 64          # one 128-byte tap per k-block needs 64-channel multiples
        w1 = torch.zeros(C1p, 1, kt1, kf1, device=c1.weight.device)
        w1[:C1] = c1.weight.detach().float()
        b1 = torch.zeros(C1p, device=c1.weight.device)
        b1[:C1] = c1.bias.detach().float()
        w2 = torch.zeros(C2, kt2, kf2, C1p, device=c1.weight.device)
        w2[..., :C1] = c2.weight.detach().float().permute(0, 2, 3, 1)   # [C2,kh,kw,C1]: k = (kh*kf2+kw)*C1 + c
        # reference feature index is c*F2 + f (conv.py:145); conv2 kernel emits f*C2 + c -> permute columns once
        wo = self.output_layer.weight.detach().float().view(self.output_size, C2, F2).permute(0, 2, 1)
        pk = {'w1': w1.contiguous(), 'b1': b1.contiguous(), 'C1p': C1p,
              'w2': w2.reshape(C2, kt2 * kf2 * C1p).to(BF16).contiguous(), 'b2': c2.bias.detach().float().contiguous(),
              'wo': wo.reshape(self.output_size, F2 * C2).to(BF16).contiguous(), 'bo': _b(self.output_layer)}
        if self.front_end_layer_norm:
            pk['ln'] = _ln(self.layer_norm)
        return pk

    def sizes(self, T):
        """[(T1, F1), (T2, F2)] for T input frames (ValueError when too short)."""
        return conv_frontend_geometry(self.layers, T, self.input_size)['sizes']

    def output_length(self, T):
        """T input frames -> T' output frames."""
        return self.sizes(T)[1][0]

    def input_window(self):
        """(stride, width): output frame t sees input frames [stride t, stride t + width) (the convolutions do not pad in
        time): (4, 7) for two 3x3 stride-2 layers."""
        return conv_frontend_geometry(self.layers)['window']

    def output_mask(self, mask):
        # Conv2dLayer.return_output_mask per layer (frontend/conv.py:78-83): mask[:, kt//2::st][:, :t]
        g = conv_frontend_geometry(self.layers, mask.shape[1], self.input_size)
        for (start, step), (t, _) in zip(g['mask'], g['sizes']):
            mask = mask[:, start::step][:, :t]
        return mask

    def training_pack(self, bf16):
        """The operands of a training pass: the inference layout, built afresh, and the transposes of w2 and wo that the
        backward's dgrad GEMMs take.  bf16 is not used: these weights are padded and permuted in fp32."""
        pk = self._build_pack()
        pk['w2_t'] = pk['w2'].t().contiguous()           # [kt2*kf2*C1p, C2]
        pk['wo_t'] = pk['wo'].t().contiguous()           # [F2*C2, D]
        return pk

    def rows_bf16(self, x, pk, posenc_scale=None, posenc_table=None, keep=False):
        """The forward of recognition and training: x f32 [B,T,F] -> (bf16 [B*T', D], T', saved).  pk: the inference pack
        or training_pack().  When posenc_* are given, x*scale+PE is fused into the Linear epilogue (pos.py:56), or applied
        after front_end_layer_norm, so the encoder can skip its own positional-encoding pass.  saved: what backward reads
        when keep, else None."""
        B, T, F = x.shape
        if F != self.input_size:
            raise ValueError(f'expected {self.input_size} features, got {F}')
        x = x.contiguous().float()
        T2 = self.output_length(T)
        h1 = ops.conv1_relu(x, pk['w1'], pk['b1'], geom=self.geom)
        h2 = ops.conv2_relu(h1, pk['w2'], pk['b2'], B, T, F, geom=self.geom)     # [B*T2, F2*C2]
        y_ln = None     # the Linear's output under front_end_layer_norm, kept for its backward
        if posenc_table is not None and not self.front_end_layer_norm:
            y = ops.linear(h2, pk['wo'], pk['bo'], EPI_TABLE, alpha=posenc_scale, table=posenc_table, period=T2)
        else:
            y = ops.linear(h2, pk['wo'], pk['bo'], EPI_BIAS)
            if self.front_end_layer_norm:
                y_ln, y = y, ops.layernorm(y, *pk['ln'])
            if posenc_table is not None:
                y = ops.scale_add_table(y, posenc_scale, posenc_table, T2)
        saved = {'x': x, 'h1': h1, 'h2': h2, 'y_ln': y_ln, 'scale': posenc_scale} if keep else None
        return y, T2, saved

    def backward(self, dx, pk, saved, g):
        """Backward of rows_bf16 from dx, the gradient of its output (bf16 [B*T', D]): x = (h2 Wo^T + bo) * scale + PE
        (without posenc: h2 Wo^T + bo) -> conv2 (implicit-GEMM forward, im2col GEMMs backward) -> conv1.  pk: the
        training_pack().  The parameter gradients go into g (train.Grads) under their names in the model ('frontend.*'), in
        the reference's layouts: output_layer's columns back in c*F2 + f order, the C1p channel padding cut off."""
        acc = g.sink is not None
        x, h1, h2 = saved['x'], saved['h1'], saved['h2']
        B, T, F = x.shape
        (T2, F2) = self.sizes(T)[1]
        C1p, C2, C1 = pk['C1p'], pk['w2'].shape[0], self.conv1.conv_layer.out_channels
        kt1, kf1, _, _, kt2, kf2, _, _ = self.geom
        dyl = ops.scale_add_table(dx, saved['scale']) if saved['scale'] is not None else dx   # d(h2 Wo^T + bo) = scale * dx
        if saved['y_ln'] is not None:                                                         # through front_end_layer_norm
            wname, bname = 'frontend.layer_norm.weight', 'frontend.layer_norm.bias'
            dyl, g[wname], g[bname] = ops.layernorm_bwd(dyl, saved['y_ln'], pk['ln'][0], dgamma=g.out(wname),
                                                        dbeta=g.out(bname), accumulate=acc)
        D_out = self.output_size
        dwo = ops.linear_wgrad(dyl, h2)                                               # [D, F2*C2], feature index f*C2 + c
        g.put('frontend.output_layer.weight', dwo.view(D_out, F2, C2).permute(0, 2, 1).reshape(D_out, C2 * F2))
        g['frontend.output_layer.bias'] = ops.colsum(dyl, out=g.out('frontend.output_layer.bias'), accumulate=acc)
        dh2 = ops.linear(dyl, pk['wo_t'])                                             # [B*T2, F2*C2]
        dpre2 = ops.relu_bwd(dh2, h2).view(B * T2 * F2, C2)
        col = ops.conv_im2col(h1, B, T, F, C1p, geom=self.geom)
        dw2 = ops.linear_wgrad(dpre2, col)                                            # [C2, kt2*kf2*C1p], k = (kh*kf2+kw)*C1p + c
        g.put('frontend.conv2.conv_layer.weight', dw2.view(C2, kt2, kf2, C1p)[..., :C1].permute(0, 3, 1, 2))
        g['frontend.conv2.conv_layer.bias'] = ops.colsum(dpre2, out=g.out('frontend.conv2.conv_layer.bias'), accumulate=acc)
        dcol = ops.linear(dpre2, pk['w2_t'])                                          # [B*T2*F2, kt2*kf2*C1p]
        del col
        dpre1 = ops.conv_col2im_relu(dcol, h1, B, T, F, C1p, geom=self.geom)
        g1 = ops.conv1_wgrad(dpre1, x, B, T, F, C1p, geom=self.geom)                  # [C1p, kt1*kf1 taps + bias]
        g.put('frontend.conv1.conv_layer.weight', g1[:C1, :kt1 * kf1].reshape(C1, 1, kt1, kf1))
        g.put('frontend.conv1.conv_layer.bias', g1[:C1, kt1 * kf1])

    def forward_bf16(self, x, posenc_scale=None, posenc_table=None):
        """x f32 [B,T,F] -> (bf16 [B*T', D], T'): rows_bf16 on the inference pack."""
        _no_train(self)
        return self.rows_bf16(x, self._pack.get(), posenc_scale, posenc_table)[:2]

    def forward(self, x, mask):
        y, T2 = self.forward_bf16(x)
        return y.float().view(x.shape[0], T2, self.output_size), self.output_mask(mask)

    def inference(self, x, mask, cache):
        y, m = self.forward(x, mask)
        return y, m, cache


class ConcatFeatureFrontEnd(nn.Module):
    """Low-frame-rate input (frontend/concat.py:11-43): output frame i stacks the n = left_frames + 1 + right_frames input
    frames from i * stride, stride = int(frame_rate / 10), frame-major (feature j * F + f, nn.Unfold's order); the input is
    zero-padded at the end so that (T_p - n) is a multiple of the stride.  No parameters.
    forward(x f32 [B,T,F], mask bool [B,T]) -> (f32 [B,T',n F], bool [B,T']).

    What the reference cannot run is refused with ValueError before any device work: right_frames >= stride (its mask
    and output lengths then differ for every T), frame_rate < 10 (stride 0) and, per call, T_p < n (nn.Unfold fails)."""

    def __init__(self, input_size, left_frames, right_frames, frame_rate=30):
        super().__init__()
        self.left_frames, self.right_frames, self.frame_rate = left_frames, right_frames, frame_rate
        self.stride = int(frame_rate / 10)
        self.input_size = input_size
        self.nframes = left_frames + right_frames + 1
        self.output_size = self.nframes * input_size
        self._pack = _Packed(self, self._build_pack)
        if frame_rate < 10:
            raise ValueError(f'concat front end: frame_rate {frame_rate} gives stride int(frame_rate / 10) = 0; it must be >= 10')
        if left_frames < 0 or right_frames < 0:
            raise ValueError('concat front end: left_frames and right_frames must be >= 0')
        if right_frames >= self.stride:
            raise ValueError(f'concat front end: right_frames {right_frames} must be less than the stride {self.stride}: the '
                             'reference\'s output mask (mask[:, left_frames::stride]) is longer than its output otherwise')

    def _padded(self, T):
        """T -> T_p, the length after the reference's zero padding (concat.py:27-30), refused where nn.Unfold fails."""
        n, s = self.nframes, self.stride
        Tp = T + (s - (T - n) % s) % s
        if Tp < n:
            raise ValueError(f'concat front end: {T} input frames pad to {Tp}, fewer than the {n} frames one output stacks')
        return Tp

    def output_length(self, T):
        """T input frames -> T' = (T_p - n) // stride + 1 output frames."""
        return (self._padded(T) - self.nframes) // self.stride + 1

    def input_window(self):
        """(stride, width): output frame t stacks input frames [stride t, stride t + n)."""
        return self.stride, self.nframes

    def output_mask(self, mask):
        """The input mask padded with False to T_p, then [:, left_frames::stride] (concat.py:29,38)."""
        B, T = mask.shape
        pad = self._padded(T) - T
        if pad:
            mask = torch.cat([mask, torch.zeros(B, pad, dtype=mask.dtype, device=mask.device)], dim=1)
        return mask[:, self.left_frames::self.stride]

    def _build_pack(self, bf16=None):
        return {}

    def training_pack(self, bf16):
        """The operands of a training pass, laid out as the inference pack.  bf16: a parameter -> its bf16 copy."""
        return self._build_pack(bf16)

    def rows_bf16(self, x, pk, posenc_scale=None, posenc_table=None, keep=False):
        """The forward of recognition and training: x f32 [B,T,F] -> (bf16 [B*T', W], T', None), W = n F rounded up to 8
        (zero columns past n F).  When posenc_* are given, x*scale+PE is applied in the same pass (otb_frame_stack's
        epilogue).  No parameters: pk is empty, and backward needs nothing saved."""
        B, T, F = x.shape
        if F != self.input_size:
            raise ValueError(f'expected {self.input_size} features, got {F}')
        T2 = self.output_length(T)
        alpha = 1.0 if posenc_table is None else posenc_scale
        return ops.frame_stack(x.contiguous().float(), self.nframes, self.stride, T2, alpha, posenc_table), T2, None

    def backward(self, dx, pk, saved, g):
        """The reference stacks without gradient (concat.py:35-37), and there are no parameters: nothing to do."""

    def forward_bf16(self, x, posenc_scale=None, posenc_table=None):
        """x f32 [B,T,F] -> (bf16 [B*T', W], T'): rows_bf16."""
        return self.rows_bf16(x, self._pack.get(), posenc_scale, posenc_table)[:2]

    def forward(self, x, mask):
        m = self.output_mask(mask)
        y, T2 = self.forward_bf16(x)
        return y[:, :self.output_size].float().view(x.shape[0], T2, self.output_size), m

    def inference(self, x, mask, cache):
        """(x, mask, cache) -> (y, mask', cache), as ConvFrontEnd.inference; the reference's BaseFrontEnd.inference takes
        no cache, so its recognizer cannot run these front ends (DESIGN.md 6)."""
        y, m = self.forward(x, mask)
        return y, m, cache


class ConcatWithLinearFrontEnd(ConcatFeatureFrontEnd):
    """ConcatFeatureFrontEnd + Linear(n F, output_size) (frontend/concat.py:46-56).  Keys: linear.weight / linear.bias.
    As in the reference, the attribute output_size stays n F (the stacked width); the Linear's own width is
    linear.out_features.  The stacked rows (bf16, K padded to a multiple of 8) feed the wgmma GEMM, whose epilogue also
    applies x*sqrt(d)+PE when the encoder lets it.  dropout > 0 is refused: the reference applies it in eval mode too
    (F.dropout with training left True, concat.py:55)."""

    def __init__(self, input_size, output_size, left_frames, right_frames, frame_rate=30, dropout=0.0):
        super().__init__(input_size, left_frames, right_frames, frame_rate)
        if dropout:
            raise NotImplementedError('concat-with-linear front end: dropout > 0 (the reference applies it in eval mode too, '
                                      'concat.py:55); use dropout 0.0')
        self.linear = nn.Linear(self.output_size, output_size)
        self.dropout = dropout

    def _build_pack(self, bf16=None):
        """{'w': the Linear weight bf16 [D, n F] as the GEMM takes it, K zero-padded to the stacked rows' width, 'b': its
        fp32 bias}.  bf16: a parameter -> its bf16 copy (a cast by default)."""
        w = bf16(self.linear.weight) if bf16 is not None else _w(self.linear)
        K = (self.output_size + 7) // 8 * 8
        if K != w.shape[1]:
            wp = torch.zeros(w.shape[0], K, dtype=BF16, device=w.device)
            wp[:, :w.shape[1]] = w
            w = wp
        return {'w': w.contiguous(), 'b': _b(self.linear)}

    def rows_bf16(self, x, pk, posenc_scale=None, posenc_table=None, keep=False):
        """The forward of recognition and training: x f32 [B,T,F] -> (bf16 [B*T', D], T', saved).  pk: the inference pack
        or training_pack().  When posenc_* are given, x*scale+PE is fused into the Linear epilogue.  saved: what backward
        reads when keep, else None."""
        stack, T2, _ = super().rows_bf16(x, pk)
        if posenc_table is not None:
            y = ops.linear(stack, pk['w'], pk['b'], EPI_TABLE, alpha=posenc_scale, table=posenc_table, period=T2)
        else:
            y = ops.linear(stack, pk['w'], pk['b'], EPI_BIAS)
        return y, T2, {'stack': stack, 'scale': posenc_scale} if keep else None

    def backward(self, dx, pk, saved, g):
        """Backward of rows_bf16 from dx, the gradient of its output (bf16 [B*T', D]): the Linear's gradients into g
        (train.Grads) as 'frontend.linear.*', the padding columns cut off.  The stacking has no gradient (concat.py:35-37)."""
        dy = ops.scale_add_table(dx, saved['scale']) if saved['scale'] is not None else dx
        g.put('frontend.linear.weight', ops.linear_wgrad(dy, saved['stack'])[:, :self.output_size])
        g['frontend.linear.bias'] = ops.colsum(dy, out=g.out('frontend.linear.bias'), accumulate=g.sink is not None)

    def forward_bf16(self, x, posenc_scale=None, posenc_table=None):
        """x f32 [B,T,F] -> (bf16 [B*T', D], T'): rows_bf16 on the inference pack."""
        _no_train(self)
        return self.rows_bf16(x, self._pack.get(), posenc_scale, posenc_table)[:2]

    def forward(self, x, mask):
        m = self.output_mask(mask)
        y, T2 = self.forward_bf16(x)
        return y.float().view(x.shape[0], T2, -1), m


# ------------------------------------------------------------------------------------------------
# parameter holders shared by encoder / decoder layers
# ------------------------------------------------------------------------------------------------
def _check_heads(d_model, n_heads):
    """The attention kernels are built for 64- and 96-wide heads (the Transformer and Conformer configs)."""
    if d_model % n_heads or d_model // n_heads not in ops.HEAD_DIMS:
        raise NotImplementedError(f'the sm_90a attention kernels support head widths d_k in {ops.HEAD_DIMS}; '
                                  f'd_model {d_model} / {n_heads} heads is not one of them')


class MultiHeadedSelfAttention(nn.Module):
    """Keys: qvk_proj.{weight,bias} [3d,d] (split order Q,K,V -- attention.py:73), output_proj.*"""

    def __init__(self, n_heads, d_model, dropout_rate=0.0, share_qvk_proj=False):
        super().__init__()
        if share_qvk_proj:
            raise NotImplementedError('share_qvk_proj')
        _check_heads(d_model, n_heads)
        self.qvk_proj = nn.Linear(d_model, d_model * 3)
        self.output_proj = nn.Linear(d_model, d_model)


class MultiHeadedCrossAttention(nn.Module):
    """Keys: q_proj.*, vk_proj.* [2d,mem] (split order K,V -- attention.py:134), output_proj.*"""

    def __init__(self, n_heads, d_model, memory_dim, dropout_rate=0.0, share_vk_proj=False):
        super().__init__()
        if share_vk_proj:
            raise NotImplementedError('share_vk_proj')
        _check_heads(d_model, n_heads)
        self.q_proj = nn.Linear(d_model, d_model)
        self.vk_proj = nn.Linear(memory_dim, d_model * 2)
        self.output_proj = nn.Linear(d_model, d_model)


class PositionwiseFeedForward(nn.Module):
    """Keys: w_1.* [d_ff or 2*d_ff, d], w_2.* [d, d_ff]   (module/ffn.py:24-41)"""

    def __init__(self, d_model, d_ff, dropout, activation='relu'):
        super().__init__()
        assert activation in ['relu', 'gelu', 'glu', 'tanh', 'swish']
        self.activation = activation
        self.w_1 = nn.Linear(d_model, d_ff * 2 if activation == 'glu' else d_ff)
        self.w_2 = nn.Linear(d_ff, d_model)


class PositionalEncoding(nn.Module):
    """module/pos.py:11-28.  Quirk kept (SURVEY.md 8a): callers pass pos_dropout into the
    ``scale_learnable`` slot, so a non-zero pos_dropout creates ``alpha`` and switches to x + alpha*PE."""

    def __init__(self, emb_dim, scale_learnable=False, dropout=0.0):
        super().__init__()
        self.emb_dim = emb_dim
        self.xscale = math.sqrt(emb_dim)
        self.scale_learnable = bool(scale_learnable)
        if self.scale_learnable:
            self.alpha = nn.Parameter(torch.tensor(1.0))

    def scale_and_table(self, n_pos, device):
        table = ops.sinusoid_table(n_pos, self.emb_dim, 0, device)
        if self.scale_learnable:
            return 1.0, table * self.alpha.detach().float()
        return self.xscale, table


def _ffn(x, pk, resid, ln=None, alpha=1.0):
    """w_2(act(w_1(x))) with the residual (and post-LayerNorm) fused into the second GEMM."""
    h = ops.linear(x, pk['w1'], pk['b1'], pk['act'])
    if ln is not None and pk['w2'].shape[0] in (64, 128, 256):
        return ops.linear(h, pk['w2'], pk['b2'], EPI_RESID_LN, resid=resid, gamma=ln[0], beta=ln[1])
    y = ops.linear(h, pk['w2'], pk['b2'], EPI_RESID, resid=resid, alpha=alpha)
    return ops.layernorm(y, *ln) if ln is not None else y


def _proj_resid_ln(ctx, w, b, resid, ln):
    """output_proj + residual (+ post-LayerNorm) in one GEMM when the row fits one tile."""
    if ln is not None and w.shape[0] in (64, 128, 256):
        return ops.linear(ctx, w, b, EPI_RESID_LN, resid=resid, gamma=ln[0], beta=ln[1])
    y = ops.linear(ctx, w, b, EPI_RESID, resid=resid)
    return ops.layernorm(y, *ln) if ln is not None else y


def _self_attn(y, resid, p, H, B, T, lengths, causal=False, ln=None, attn_sink=None, context=None):
    """resid + output_proj(MHA(y)) (+ LayerNorm): QKV GEMM -> fused attention -> output projection with the residual.
    attn_sink (a list): the attention weights f32 [B, H, T, T] are appended to it.  context(qkv) -> bf16 [rows, d]: the
    attention context of a KV-cached step (the newest position of each row against its cached prefix) instead of the
    attention over the rows of this call."""
    d = y.shape[1]
    qkv = ops.linear(y, p['wqkv'], p['bqkv'])
    if context is not None:
        return _proj_resid_ln(context(qkv), p['wo'], p['bo'], resid, ln)
    if attn_sink is not None:
        attn_sink.append(ops.attention_probs(qkv, qkv, B, H, T, T, kv_len=lengths, causal=causal, q_col0=0, k_col0=d, d_k=d // H))
    ctx = ops.attention(qkv, qkv, qkv, B, H, T, T, kv_len=lengths, causal=causal, q_col0=0, k_col0=d, v_col0=2 * d,
                        d_k=d // H)
    return _proj_resid_ln(ctx, p['wo'], p['bo'], resid, ln)


def _ffn_pack(ff):
    return {'w1': _w(ff.w_1), 'b1': _b(ff.w_1), 'w2': _w(ff.w_2), 'b2': _b(ff.w_2),
            'act': ACT_EPILOGUE[ff.activation]}


def encoder_attn_weights(n_blocks, sink):
    """The encoders' attn_weights dict (encoder/transformer.py:126-129): the maps collected in sink, or None maps."""
    return {'enc_block_%d' % i: {'slf_attn_weights': sink[i] if sink is not None else None} for i in range(n_blocks)}


# ------------------------------------------------------------------------------------------------
# encoder
# ------------------------------------------------------------------------------------------------
class TransformerEncoderLayer(nn.Module):
    def __init__(self, n_heads, d_model, d_ff, slf_attn_dropout, ffn_dropout, residual_dropout,
                 normalize_before=False, concat_after=False, relative_positional=False, activation='relu'):
        super().__init__()
        if concat_after:
            raise NotImplementedError('concat_after is not used by any shipped config')
        self.n_heads = n_heads
        self.normalize_before = normalize_before
        self.relative_positional = relative_positional
        # dropout is a training-time op (encoder/transformer.py:32-33,54,61); inference ignores it, train.py checks it
        self.dropout_rates = {'slf_attn_dropout': slf_attn_dropout, 'ffn_dropout': ffn_dropout,
                              'residual_dropout': residual_dropout}
        if relative_positional:     # encoder/transformer.py:23-24: Transformer-XL style attention, NO output projection (SURVEY 8a quirk)
            self.slf_attn = MultiHeadedSelfAttentionWithRelPos(n_heads, d_model, slf_attn_dropout)
        else:
            self.slf_attn = MultiHeadedSelfAttention(n_heads, d_model, slf_attn_dropout)
        self.feed_forward = PositionwiseFeedForward(d_model, d_ff, ffn_dropout, activation)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)

    def pack(self):
        a = self.slf_attn
        pk = {'ffn': _ffn_pack(self.feed_forward), 'ln1': _ln(self.norm1), 'ln2': _ln(self.norm2)}
        if self.relative_positional:
            pk['rel'] = a.pack()
        else:
            pk.update({'wqkv': _w(a.qvk_proj), 'bqkv': _b(a.qvk_proj), 'wo': _w(a.output_proj), 'bo': _b(a.output_proj)})
        return pk

    def run(self, x, pk, B, T, lengths, causal=False, pos_bf16=None, attn_sink=None, context=None):
        """x bf16 [B*T, d] -> bf16 [B*T, d]   (encoder/transformer.py:41-65); causal=True is the tril mask the
        Transformer LM feeds to the same layer (model/lm.py:14-18,148-151).  attn_sink, context: see _self_attn (the
        Transformer LM's KV-cached step passes context)."""
        nb = self.normalize_before
        if nb:
            x = ops.layernorm(x, *pk['ln1'])          # residual is taken AFTER the norm (transformer.py:42-44)
        ln = None if nb else pk['ln1']
        if self.relative_positional:
            if causal or context is not None:
                raise NotImplementedError('causal rel-pos attention')
            x = self.slf_attn.run(x, x, pk['rel'], B, T, lengths, pos_bf16, attn_sink)   # x + attention (no output projection)
            if ln is not None:
                x = ops.layernorm(x, *ln)
        else:
            x = _self_attn(x, x, pk, self.n_heads, B, T, lengths, causal, ln, attn_sink, context)
        if nb:
            x = ops.layernorm(x, *pk['ln2'])
        return _ffn(x, pk['ffn'], x, None if nb else pk['ln2'])


class _SpeechEncoder(nn.Module):
    """The positional input and module-level forward that TransformerEncoder and ConformerEncoder share.  Abs-pos encoders
    scale their input and add PE (pos.py:56); rel-pos encoders take it as it is and give PE[-(T-1)..T-1] to their
    attention (encoder/transformer.py:116-119, encoder/conformer.py:140-149)."""

    def fuse_abs_posenc(self):
        """True when x*scale+PE may be fused into the front end's last kernel."""
        return self.positional_encoding and not self.relative_positional

    def rel_pos_table(self, T, device):
        """PE[-(T-1) .. T-1] bf16 [2T-1, d], the GEMM operand of the rel-pos attention's pos_proj (cached per T and device);
        None for an encoder without rel-pos attention."""
        if not (self.positional_encoding and self.relative_positional):
            return None
        key = (T, device.index)
        p = self._pos_cache.get(key)
        if p is None:
            p = ops.scale_add_table(ops.sinusoid_table(2 * T - 1, self.d_model, -(T - 1), device))
            self._pos_cache[key] = p
        return p

    def apply_posenc_bf16(self, x, B, T):
        if self.fuse_abs_posenc():
            scale, table = self.pos_emb.scale_and_table(T, x.device)
            return ops.scale_add_table(x, scale, table, T)
        return x if x.dtype == BF16 else ops.scale_add_table(x)

    def forward(self, inputs, mask):
        B, T, D = inputs.shape
        x = self.apply_posenc_bf16(inputs.contiguous().view(B * T, D), B, T)
        sink = [] if self.return_attn_weights else None
        y = self.forward_bf16(x, B, T, _lengths(mask), sink)
        return y.float().view(B, T, D), mask, encoder_attn_weights(len(self.blocks), sink)


def encoder_input_bf16(frontend, encoder, x, mask, pk, keep=False):
    """The front half of a speech model, for recognition and training: x f32 [B,T,F], mask bool [B,T] -> (the encoder's
    input bf16 [B*T', d], lengths i32 [B], T', what frontend.backward reads when keep).  An abs-pos encoder's x*scale+PE is
    fused into the front end; a rel-pos encoder takes the front end's rows as they are.  pk: the front end's operands."""
    T2 = frontend.output_length(x.shape[1])
    lengths = _lengths(frontend.output_mask(mask))
    scale, table = encoder.pos_emb.scale_and_table(T2, x.device) if encoder.fuse_abs_posenc() else (None, None)
    y, _, saved = frontend.rows_bf16(x, pk, scale, table, keep)
    return y, lengths, T2, saved


class TransformerEncoder(_SpeechEncoder):
    """forward(inputs f32 [B,T,D], mask bool [B,T]) -> (f32 [B,T,D], mask, attn_weights)

    ``attn_weights`` maps 'enc_block_i' -> {'slf_attn_weights': P}.  The fused attention kernel never forms P, so by
    default P is None; with ``return_attn_weights = True`` it is the reference's f32 [B, h, T, T] softmax
    (encoder/transformer.py:126-129), written by one extra kernel per block (otb_attention_probs).  The encoder output
    is the same either way.
    """

    def __init__(self, d_model=256, n_heads=4, d_ff=2048, n_blocks=6, pos_dropout=0.0, slf_attn_dropout=0.0,
                 ffn_dropout=0.0, residual_dropout=0.1, normalize_before=False, concat_after=False,
                 relative_positional=False, activation='relu'):
        super().__init__()
        self.d_model = d_model
        self.normalize_before = normalize_before
        self.positional_encoding = True     # ConformerEncoder's switch: the reference's Transformer encoder always has one
        self.relative_positional = relative_positional
        self.pos_emb = PositionalEncoding(d_model, pos_dropout)
        self.blocks = nn.ModuleList([
            TransformerEncoderLayer(n_heads, d_model, d_ff, slf_attn_dropout, ffn_dropout, residual_dropout,
                                    normalize_before, concat_after, relative_positional, activation)
            for _ in range(n_blocks)])
        if normalize_before:
            self.norm = nn.LayerNorm(d_model)
        self._pack = _Packed(self, lambda: {'blocks': [b.pack() for b in self.blocks],
                                            'norm': _ln(self.norm) if normalize_before else None})
        self._pos_cache = {}
        self.return_attn_weights = False

    def forward_bf16(self, x, B, T, lengths, attn_sink=None):
        """x bf16 [B*T, d] with the positional encoding already applied (abs-pos) / the raw front-end output (rel-pos).
        attn_sink (a list): each block's attention weights f32 [B, H, T, T] are appended to it."""
        _no_train(self)
        pk = self._pack.get()
        pos = self.rel_pos_table(T, x.device)
        for blk, bpk in zip(self.blocks, pk['blocks']):
            x = blk.run(x, bpk, B, T, lengths, pos_bf16=pos, attn_sink=attn_sink)
        if self.normalize_before:
            x = ops.layernorm(x, *pk['norm'])
        return x


# ------------------------------------------------------------------------------------------------
# Conformer encoder  (otrans/encoder/conformer.py, otrans/module/conformer.py, attention.py:176-257)
# ------------------------------------------------------------------------------------------------
class MultiHeadedSelfAttentionWithRelPos(nn.Module):
    """Keys: qvk_proj.*, pos_proj.weight, posu, posv  (attention.py:176-194).  Quirk kept (SURVEY.md 8a): the
    reference passes dropout_rate into the enable_output_proj slot, so with the shipped slf_attn_dropout 0.0
    there is NO output projection; a non-zero rate makes the reference itself crash."""

    def __init__(self, n_heads, d_model, dropout_rate=0.0, skip_term_b=False, share_qvk_proj=False):
        super().__init__()
        if dropout_rate or skip_term_b or share_qvk_proj:
            raise NotImplementedError('rel-pos attention: dropout / skip_term_b / share_qvk_proj')
        _check_heads(d_model, n_heads)
        self.nheads, self.d_model = n_heads, d_model
        self.qvk_proj = nn.Linear(d_model, d_model * 3)
        self.pos_proj = nn.Linear(d_model, d_model, bias=False)
        self.posu = nn.Parameter(torch.Tensor(1, 1, n_heads, d_model // n_heads))
        self.posv = nn.Parameter(torch.Tensor(1, 1, n_heads, d_model // n_heads))
        torch.nn.init.xavier_normal_(self.posu)
        torch.nn.init.xavier_normal_(self.posv)

    def pack(self):
        d = self.d_model
        w, b = self.qvk_proj.weight.detach().float(), self.qvk_proj.bias.detach().float()
        u, v = self.posu.detach().float().reshape(d), self.posv.detach().float().reshape(d)
        # one projection producing [q+u | q+v | k | v]: (q+u) = x Wq^T + (bq + u)
        w_ext = torch.cat([w[:d], w[:d], w[d:2 * d], w[2 * d:]], 0)
        b_ext = torch.cat([b[:d] + u, b[:d] + v, b[d:2 * d], b[2 * d:]], 0)
        return {'wext': w_ext.to(BF16).contiguous(), 'bext': b_ext.contiguous(), 'wpos': _w(self.pos_proj)}

    def run(self, y, x_resid, pk, B, T, lengths, pos_bf16, attn_sink=None):
        """y = LN(x) bf16 [B*T,d]; returns x_resid + attention (no output projection).  attn_sink (a list): the attention
        weights f32 [B, H, T, T] are appended to it."""
        d, H = self.d_model, self.nheads
        ext = ops.linear(y, pk['wext'], pk['bext'])                       # [M, 4d]
        pproj = ops.linear(pos_bf16, pk['wpos'])                          # [2T-1, d]  pos_proj(PE[-(T-1)..T-1])
        bd = rel_pos_band(ext, pproj, H, B, T)
        if attn_sink is not None:   # scores (q+u) k^T + BD, as the fused kernel below forms them
            attn_sink.append(ops.attention_probs(ext, ext, B, H, T, T, kv_len=lengths, q_col0=0, k_col0=2 * d, bd=bd, d_k=d // H))
        return ops.attention(ext, ext, ext, B, H, T, T, kv_len=lengths, q_col0=0, k_col0=2 * d, v_col0=3 * d,
                             bd=bd, resid=x_resid, d_k=d // H)


def rel_pos_band(ext, pproj, H, B, T):
    """BD f32 [H, B*T, ld]: row i of head h holds (q_i+v)_h . P_h[m] for m = 0 .. 2T-2 (the attention kernels read the
    j-i+T-1 diagonal band).  ext = [q+u | q+v | k | v] bf16 [B*T, 4d]; pproj = pos_proj(PE[-(T-1)..T-1]) bf16 [2T-1, d]."""
    d = ext.shape[1] // 4
    dk = d // H
    ld = (2 * T - 1 + 3) // 4 * 4
    bd = torch.empty(H, B * T, ld, dtype=torch.float32, device=ext.device)
    for h in range(H):  # BD_full[h] = (q+v)_h P_h^T
        ops.linear(ext[:, d + dk * h: d + dk * (h + 1)], pproj[:, dk * h: dk * (h + 1)], out=bd[h])
    return bd


class ConformerConvolutionModule(nn.Module):
    """Keys: pointwise_conv1.*, depthwise_conv.*, batch_norm.*, pointwise_conv2.*  (module/conformer.py:12-34)."""

    def __init__(self, channels, kernel_size, bias=True, dropout=0.0):
        super().__init__()
        assert kernel_size % 2 == 1
        self.pointwise_conv1 = nn.Linear(channels, 2 * channels, bias=bias)
        self.depthwise_conv = nn.Conv1d(channels, channels, kernel_size, stride=1, padding=(kernel_size - 1) // 2,
                                        groups=channels, bias=bias)
        self.batch_norm = nn.BatchNorm1d(channels)
        self.pointwise_conv2 = nn.Linear(channels, channels, bias=bias)

    def pack(self):
        bn, dw = self.batch_norm, self.depthwise_conv
        s = bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)
        w = dw.weight.detach().float()[:, 0, :] * s[:, None]                       # [C,k] BN scale folded in
        b0 = dw.bias.detach().float() if dw.bias is not None else torch.zeros_like(s)
        b = (b0 - bn.running_mean.detach().float()) * s + bn.bias.detach().float()
        return {'w1': _w(self.pointwise_conv1), 'b1': _b(self.pointwise_conv1),
                'wd': w.t().contiguous(), 'bd': b.contiguous(),                     # tap-major [k,C]
                'w2': _w(self.pointwise_conv2), 'b2': _b(self.pointwise_conv2)}

    def run(self, y, x_resid, pk, B, T, lengths):
        """x_resid + conv_module(y); padded frames are zeroed after the GLU and after the last Linear
        (module/conformer.py:46,55) through the GEMM's row mask."""
        g = ops.linear(y, pk['w1'], pk['b1'], EPI_GLU, row_len=lengths, row_period=T)
        c = ops.dwconv_swish(g, pk['wd'], pk['bd'], B, T)
        return ops.linear(c, pk['w2'], pk['b2'], EPI_RESID, resid=x_resid, row_len=lengths, row_period=T)


class ConformerEncoderBlock(nn.Module):
    def __init__(self, d_model, d_ff, cov_kernel_size, n_heads, slf_attn_dropout=0.0, ffn_dropout=0.0,
                 residual_dropout=0.1, conv_dropout=0.0, macaron_style=True, conv_first=False, ffn_scale=0.5,
                 conv_bias=True, relative_positional=True, activation='glu'):
        super().__init__()
        self.conv_first, self.macaron_style, self.ffn_scale = conv_first, macaron_style, ffn_scale
        self.relative_positional, self.n_heads = relative_positional, n_heads
        # training-time rates (encoder/conformer.py:53-72); inference ignores them, train.py checks them.  conv_dropout builds
        # a Dropout the reference never applies (module/conformer.py:34,36-57).
        self.dropout_rates = {'slf_attn_dropout': slf_attn_dropout, 'ffn_dropout': ffn_dropout,
                              'residual_dropout': residual_dropout, 'conv_dropout': conv_dropout}
        self.conv_bias = conv_bias
        if macaron_style:
            self.pre_ffn = PositionwiseFeedForward(d_model, d_ff, ffn_dropout, activation=activation)
            self.macaron_ffn_norm = nn.LayerNorm(d_model)
        if relative_positional:
            self.mha = MultiHeadedSelfAttentionWithRelPos(n_heads, d_model, slf_attn_dropout)
        else:
            self.mha = MultiHeadedSelfAttention(n_heads, d_model, slf_attn_dropout)
        self.mha_norm = nn.LayerNorm(d_model)
        self.conv = ConformerConvolutionModule(d_model, cov_kernel_size, conv_bias, conv_dropout)
        self.conv_norm = nn.LayerNorm(d_model)
        # kept for state_dict parity; the reference never applies post_ffn, only post_ffn_norm (conformer.py:87)
        self.post_ffn = PositionwiseFeedForward(d_model, d_ff, ffn_dropout, activation=activation)
        self.post_ffn_norm = nn.LayerNorm(d_model)
        self.final_norm = nn.LayerNorm(d_model)

    def pack(self):
        pk = {'mha_ln': _ln(self.mha_norm), 'conv_ln': _ln(self.conv_norm), 'post_ln': _ln(self.post_ffn_norm),
              'final_ln': _ln(self.final_norm), 'conv': self.conv.pack()}
        if self.macaron_style:
            pk['pre_ffn'] = _ffn_pack(self.pre_ffn)
            pk['mac_ln'] = _ln(self.macaron_ffn_norm)
        if self.relative_positional:
            pk['mha'] = self.mha.pack()
        else:
            a = self.mha
            pk['mha'] = {'wqkv': _w(a.qvk_proj), 'bqkv': _b(a.qvk_proj), 'wo': _w(a.output_proj), 'bo': _b(a.output_proj)}
        return pk

    def _attn(self, x, pk, B, T, lengths, pos_bf16, attn_sink):
        y = ops.layernorm(x, *pk['mha_ln'])
        if self.relative_positional:
            return self.mha.run(y, x, pk['mha'], B, T, lengths, pos_bf16, attn_sink)
        return _self_attn(y, x, pk['mha'], self.n_heads, B, T, lengths, attn_sink=attn_sink)

    def _conv(self, x, pk, B, T, lengths):
        return self.conv.run(ops.layernorm(x, *pk['conv_ln']), x, pk['conv'], B, T, lengths)

    def run(self, x, pk, B, T, lengths, pos_bf16, attn_sink=None):
        """ConformerEncoderBlock.forward (encoder/conformer.py:75-89) with the residual dropout disabled.  attn_sink: see
        MultiHeadedSelfAttentionWithRelPos.run."""
        if self.macaron_style:
            y = ops.layernorm(x, *pk['mac_ln'])
            f = pk['pre_ffn']
            h = ops.linear(y, f['w1'], f['b1'], f['act'])
            x = ops.linear(h, f['w2'], f['b2'], EPI_RESID, resid=x, alpha=self.ffn_scale)
        if self.conv_first:
            x = self._attn(self._conv(x, pk, B, T, lengths), pk, B, T, lengths, pos_bf16, attn_sink)
        else:
            x = self._conv(self._attn(x, pk, B, T, lengths, pos_bf16, attn_sink), pk, B, T, lengths)
        return ops.layernorm(x, *pk['post_ln'], *pk['final_ln'])   # post_ffn_norm then final_norm, one kernel


class ConformerEncoder(_SpeechEncoder):
    """forward(inputs f32 [B,T,D], mask bool [B,T]) -> (f32 [B,T,D], mask, attn_weights)   (encoder/conformer.py:117-164)

    The reference applies F.dropout(p=residual_dropout) with training=True even in eval() (conformer.py:53,58,63,72),
    i.e. its inference is stochastic for residual_dropout > 0 (SURVEY.md 8a).  This implementation is the
    deterministic network (no dropout at inference); parity is defined against residual_dropout = 0.0.

    ``attn_weights`` as TransformerEncoder's: None maps unless ``return_attn_weights`` is set."""

    def __init__(self, d_model, d_ff, cov_kernel_size, n_heads, nblocks=12, pos_dropout=0.0, slf_attn_dropout=0.0,
                 ffn_dropout=0.0, residual_dropout=0.1, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5,
                 conv_bias=True, positional_encoding=True, relative_positional=True, conv_first=False,
                 activation='glu'):
        super().__init__()
        self.positional_encoding = positional_encoding
        self.relative_positional = relative_positional
        self.output_size = self.d_model = d_model
        if positional_encoding:
            self.pos_emb = PositionalEncoding(d_model, pos_dropout)
        self.blocks = nn.ModuleList([
            ConformerEncoderBlock(d_model, d_ff, cov_kernel_size, n_heads, slf_attn_dropout, ffn_dropout,
                                  residual_dropout, conv_dropout, macaron_style, conv_first, ffn_scale, conv_bias,
                                  relative_positional, activation) for _ in range(nblocks)])
        self._pack = _Packed(self, lambda: [b.pack() for b in self.blocks])
        self._pos_cache = {}
        self.return_attn_weights = False

    def forward_bf16(self, x, B, T, lengths, attn_sink=None):
        """attn_sink (a list): each block's attention weights f32 [B, H, T, T] are appended to it."""
        _no_train(self)
        pks = self._pack.get()
        pos = self.rel_pos_table(T, x.device)
        for blk, pk in zip(self.blocks, pks):
            x = blk.run(x, pk, B, T, lengths, pos, attn_sink)
        return x


# ------------------------------------------------------------------------------------------------
# decoder
# ------------------------------------------------------------------------------------------------
class SelfAttnCache:
    """The self-attention half of the KV caches of the incremental decoder (DecoderCache) and the Transformer LM (LMCache):
    K/V of every decoded position [layer, position, row, d], the ping-pong ancestry table anc [2, N, max_len], the device
    step counter and the positional table.  Beam pruning never moves K/V rows, it rewrites a 4-byte ancestry entry per
    (row, position): ``reorder(parent_rows)``.  The cache is tied to the weight pack its K/V were computed with.

    anc / step_ptr: a search that keeps its own ancestry and step counter (recognize.BeamDecoder's BeamState) passes them
    in, and its beam kernel reorders the cache; such a cache is never reordered from the host."""

    def __init__(self, what, pk, n_layers, n_rows, d, max_len, device, anc=None, step_ptr=None):
        self._what, self._pk = what, pk
        self.N, self.Lmax, self.step = n_rows, max_len, 0
        self.kc = torch.zeros(n_layers, max_len, n_rows, d, dtype=BF16, device=device)
        self.vc = torch.zeros(n_layers, max_len, n_rows, d, dtype=BF16, device=device)
        self.anc = torch.zeros(2, n_rows, max_len, dtype=torch.int32, device=device) if anc is None else anc
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=device) if step_ptr is None else step_ptr
        self.table = ops.sinusoid_table(max_len + 1, d, 0, device)

    def begin_step(self, pk, preds):
        """Refuse, before any device work, an incremental call that does not fit the cache (preds i64 [N, step + 1]: one
        new token per row and call), then point the device step counter at the new position."""
        name = type(self).__name__
        if pk is not self._pk:
            raise RuntimeError(f'{name} was built with different {self._what} weights (parameters changed since init_cache)')
        if preds.dim() != 2 or preds.shape[0] != self.N or preds.shape[1] != self.step + 1:
            raise ValueError(f'cached inference expects preds [N={self.N}, {self.step + 1}] (one new token per call), got {tuple(preds.shape)}')
        if self.step >= self.Lmax:
            raise ValueError(f'{name} is full (max_len reached)')
        self.step_dev.fill_(self.step)

    def reorder(self, parent_rows):
        """Row n of the next step continues row parent_rows[n] (i64/i32 [N], global row indices)."""
        if self.step == 0:
            raise RuntimeError(f'{type(self).__name__}.reorder before the first inference step')
        s = self.step - 1                     # the position that was just decoded
        cur, nxt = s & 1, (s & 1) ^ 1
        par = parent_rows.view(-1).long()
        self.anc[nxt] = self.anc[cur].index_select(0, par)
        self.anc[nxt, :, s] = par.to(torch.int32)

    def advance_without_reorder(self):
        """Greedy / teacher-forced use (no pruning): every row continues itself."""
        self.reorder(torch.arange(self.N, device=self.anc.device))


class DecoderCache(SelfAttnCache):
    """The decoder cache the reference stubbed out (decoder/transformer.py:92-126,188-203; README TODO), as the opaque
    `cache` object of ``TransformerDecoder.inference(preds, memory, memory_mask, cache)``:

      * cross-attention K/V of the memory, projected ONCE (the reference re-runs vk_proj on the beam-tiled memory at every
        step, attention.py:129).  When the memory rows are the beam-tiled copies of `batch` utterances
        (recognize/speech2text.py:51-52) pass ``beam`` so that each utterance is projected once and shared by its beams;
      * self-attention K/V of every decoded position (SelfAttnCache); ``reorder(parent_rows)`` is what `decode_step` calls
        where the reference intended reselect_hidden* (recognize/speech2text.py:195-218).

    Build it with ``TransformerDecoder.init_cache``.  One `inference` call consumes exactly one new token per row."""

    def __init__(self, decoder, memory, memory_mask, max_len, beam=1):
        n, T, D = memory.shape
        if n % beam:
            raise ValueError('DecoderCache: memory rows must be a multiple of beam')
        dev = memory.device
        nl, d = len(decoder.blocks), decoder.d_model
        pk = decoder.packed()
        super().__init__('decoder', pk, nl, n, d, max_len, dev)
        self.T, self.beam = T, beam
        self.batch = n // beam
        mem = memory.contiguous().view(self.batch, beam, T, D)[:, 0]                 # one copy per utterance
        msk = memory_mask.contiguous().view(self.batch, beam, T)[:, 0]
        mem_bf16 = ops.scale_add_table(mem.contiguous().view(self.batch * T, D).float())
        self.mem_len = _lengths(msk)
        self.kvx = torch.empty(nl, self.batch * T, 2 * d, dtype=BF16, device=dev)
        for l, p in enumerate(pk['blocks']):
            ops.linear(mem_bf16, p['wkv'], p['bkv'], out=self.kvx[l])


class TransformerDecoderLayer(nn.Module):
    def __init__(self, n_heads, d_model, d_ff, memory_dim, slf_attn_dropout=0.0, src_attn_dropout=0.0,
                 ffn_dropout=0.0, residual_dropout=0.1, normalize_before=False, concat_after=False,
                 relative_positional=False, activation='relu'):
        super().__init__()
        if concat_after or relative_positional:
            raise NotImplementedError('concat_after / relative_positional decoder')
        self.n_heads = n_heads
        self.normalize_before = normalize_before
        self.dropout_rates = {'slf_attn_dropout': slf_attn_dropout, 'src_attn_dropout': src_attn_dropout,
                              'ffn_dropout': ffn_dropout, 'residual_dropout': residual_dropout}
        self.slf_attn = MultiHeadedSelfAttention(n_heads, d_model, slf_attn_dropout)
        self.src_attn = MultiHeadedCrossAttention(n_heads, d_model, memory_dim, src_attn_dropout)
        self.feed_forward = PositionwiseFeedForward(d_model, d_ff, ffn_dropout, activation)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)
        self.norm3 = nn.LayerNorm(d_model)

    def pack(self):
        a, c = self.slf_attn, self.src_attn
        return {'wqkv': _w(a.qvk_proj), 'bqkv': _b(a.qvk_proj), 'wo': _w(a.output_proj), 'bo': _b(a.output_proj),
                'wq': _w(c.q_proj), 'bq': _b(c.q_proj), 'wkv': _w(c.vk_proj), 'bkv': _b(c.vk_proj),
                'wo2': _w(c.output_proj), 'bo2': _b(c.output_proj), 'ffn': _ffn_pack(self.feed_forward),
                'ln1': _ln(self.norm1), 'ln2': _ln(self.norm2), 'ln3': _ln(self.norm3)}


class TransformerDecoder(nn.Module):
    """forward(targets i64 [B,L], memory f32 [B,T,D], memory_mask bool [B,T]) -> (logits f32 [B,L,V], attn)
    inference(preds i64 [N,l], memory, memory_mask, cache) -> (log_probs f32 [N,V], cache, attn)
    (decoder/transformer.py:161-208).  `cache` is passed through untouched exactly like the reference;
    the KV-cached incremental path lives in recognize.BeamDecoder.

    ``attn`` maps 'dec_block_i' -> {'slf_attn_weights', 'src_attn_weights'}: None by default; with
    ``return_attn_weights = True``, forward (and inference without a DecoderCache) returns the reference's f32 maps,
    [B, h, L, L] under the causal mask and [B, h, L, T] under the memory lengths."""

    def __init__(self, vocab_size, d_model=256, n_heads=4, d_ff=2048, memory_dim=256, n_blocks=6, pos_dropout=0.0,
                 slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.1,
                 activation='relu', normalize_before=True, concat_after=False, share_embedding=False):
        super().__init__()
        self.decoder_type = 'transformer'
        self.normalize_before = normalize_before
        self.relative_positional = False
        self.d_model, self.n_heads, self.vocab_size = d_model, n_heads, vocab_size
        self.embedding = nn.Embedding(vocab_size, d_model)
        self.pos_emb = PositionalEncoding(d_model, pos_dropout)
        self.blocks = nn.ModuleList([
            TransformerDecoderLayer(n_heads, d_model, d_ff, memory_dim, slf_attn_dropout, src_attn_dropout,
                                    ffn_dropout, residual_dropout, normalize_before, concat_after, False, activation)
            for _ in range(n_blocks)])
        if normalize_before:
            self.after_norm = nn.LayerNorm(d_model)
        self.output_layer = nn.Linear(d_model, vocab_size)
        if share_embedding:
            assert self.embedding.weight.size() == self.output_layer.weight.size()
            self.output_layer.weight = self.embedding.weight   # tied (decoder/transformer.py:156-158)
        self._pack = _Packed(self, self._build_pack)
        self.return_attn_weights = False

    def _build_pack(self):
        emb = self.embedding.weight.detach().to(BF16).contiguous()
        tied = self.output_layer.weight is self.embedding.weight
        return {'emb': emb, 'wout': emb if tied else _w(self.output_layer), 'bout': _b(self.output_layer),
                'blocks': [b.pack() for b in self.blocks],
                'after': _ln(self.after_norm) if self.normalize_before else None}

    def packed(self):
        return self._pack.get()

    @property
    def ld_logits(self):
        return (self.vocab_size + 7) // 8 * 8

    def _layers(self, pk, x, self_attn, cross_attn):
        """The decoder layers (decoder/transformer.py:54-90) and the final after_norm over x bf16 [rows, d].  Only the
        attention contexts depend on the caller: self_attn(l, qkv) and cross_attn(l, q) return those of layer l."""
        nb = self.normalize_before
        for l, p in enumerate(pk['blocks']):
            if nb:
                x = ops.layernorm(x, *p['ln1'])
            qkv = ops.linear(x, p['wqkv'], p['bqkv'])
            x = _proj_resid_ln(self_attn(l, qkv), p['wo'], p['bo'], x, None if nb else p['ln1'])
            if nb:
                x = ops.layernorm(x, *p['ln2'])
            q = ops.linear(x, p['wq'], p['bq'])
            x = _proj_resid_ln(cross_attn(l, q), p['wo2'], p['bo2'], x, None if nb else p['ln2'])
            if nb:
                x = ops.layernorm(x, *p['ln3'])
            x = _ffn(x, p['ffn'], x, None if nb else p['ln3'])
        if nb:
            x = ops.layernorm(x, *pk['after'])
        return x

    def decode_cached_bf16(self, pk, x, kc, vc, anc, step_ptr, kvx, mem_len, beam, T):
        """The layers on the newest token of N = batch * beam hypotheses, x bf16 [N, d].  Self-attention reads the cached
        keys / values kc, vc [layer, position, row, d] through the ancestry table `anc`; cross-attention reads the memory's
        K|V kvx [layer, batch * T, 2d], projected once per utterance."""
        d, H, N, Lmax, batch = self.d_model, self.n_heads, x.shape[0], kc.shape[1], mem_len.shape[0]
        return self._layers(
            pk, x, lambda l, qkv: ops.decode_self_attn(qkv, kc[l], vc[l], anc, step_ptr, N, H, Lmax),
            # the `beam` hypotheses of utterance b are the query rows [b*beam, (b+1)*beam) of one attention problem
            # (the attention kernel pads the problem to 128 query rows)
            lambda l, q: ops.attention(q, kvx[l], kvx[l], batch, H, beam, T, kv_len=mem_len, k_col0=0, v_col0=d, d_k=d // H))

    def forward_bf16(self, targets, memory_bf16, mem_len, B, L, T, attn_sink=None):
        """targets i64 [B,L]; memory bf16 [B*T, D] -> logits f32 [B*L, ld_logits] (first V columns valid).
        attn_sink (a list): each layer's self- and cross-attention weights, f32 [B, H, L, L] and [B, H, L, T], are
        appended to it in that order."""
        return self.score_bf16(targets, memory_bf16, mem_len, B, 1, L, T, attn_sink)

    def score_bf16(self, inputs, memory_bf16, mem_len, B, K, Lp, T, attn_sink=None):
        """Teacher-forced logits of K sequences per utterance (the second pass of n-best rescoring): inputs i64 [B*K, Lp],
        memory bf16 [B*T, D] -> logits f32 [B*K*Lp, ld_logits] (first V columns valid).  Self-attention is causal within
        each of the B*K sequences; cross-attention treats the K*Lp query rows of utterance b as one problem against its
        memory, so the memory's K|V is projected once per utterance, not once per sequence."""
        _no_train(self)
        pk = self._pack.get()
        d, H = self.d_model, self.n_heads
        scale, table = self.pos_emb.scale_and_table(Lp, memory_bf16.device)
        if self.pos_emb.scale_learnable:
            raise NotImplementedError('decoder with learnable positional scale')
        x = ops.embed_posenc(inputs.contiguous(), pk['emb'], table, B * K * Lp, d, period=Lp)

        def self_attn(l, qkv):
            if attn_sink is not None:
                attn_sink.append(ops.attention_probs(qkv, qkv, B * K, H, Lp, Lp, causal=True, q_col0=0, k_col0=d, d_k=d // H))
            return ops.attention(qkv, qkv, qkv, B * K, H, Lp, Lp, causal=True, q_col0=0, k_col0=d, v_col0=2 * d, d_k=d // H)

        def cross_attn(l, q):       # the memory's K|V, projected per layer after the query GEMM
            p = pk['blocks'][l]
            kv = ops.linear(memory_bf16, p['wkv'], p['bkv'])
            if attn_sink is not None:
                attn_sink.append(ops.attention_probs(q, kv, B, H, K * Lp, T, kv_len=mem_len, k_col0=0, d_k=d // H))
            return ops.attention(q, kv, kv, B, H, K * Lp, T, kv_len=mem_len, k_col0=0, v_col0=d, d_k=d // H)

        x = self._layers(pk, x, self_attn, cross_attn)
        return ops.linear(x, pk['wout'], pk['bout'], EPI_BIAS, out_f32=True, n_out=self.ld_logits)

    def forward(self, targets, memory, memory_mask):
        B, L = targets.shape
        T, D = memory.shape[1], memory.shape[2]
        mem = ops.scale_add_table(memory.contiguous().view(B * T, D))   # f32 -> bf16
        sink = [] if self.return_attn_weights else None
        logits = self.forward_bf16(targets, mem, _lengths(memory_mask), B, L, T, sink)
        attn = {'dec_block_%d' % i: {'slf_attn_weights': sink[2 * i] if sink is not None else None,
                                     'src_attn_weights': sink[2 * i + 1] if sink is not None else None}
                for i in range(len(self.blocks))}
        return logits.view(B, L, -1)[:, :, :self.vocab_size], attn

    def init_cache(self, memory, memory_mask, max_len, beam=1):
        """KV cache for `inference` (see DecoderCache).  memory f32 [N,T,D] (beam-tiled or not), memory_mask bool [N,T]."""
        _no_train(self)
        return DecoderCache(self, memory, memory_mask, max_len, beam)

    def inference(self, preds, memory, memory_mask=None, cache=None):
        """decoder/transformer.py:185-208.  cache None (the reference's only working mode): the whole prefix is recomputed.
        cache = DecoderCache (``init_cache``): only the newest token preds[:, -1] is run through the layers against the cached
        keys / values -- O(l) instead of O(l^2) per step -- and the same object is returned; the caller reorders it after
        pruning (SpeechToTextRecognizer.decode_step does).  The cached path returns None maps even with
        return_attn_weights set: it never forms the attention weights of the earlier positions."""
        assert preds.dim() == 2
        if isinstance(cache, DecoderCache):
            return self._inference_cached(preds, cache)
        logits, attn = self.forward(preds, memory, memory_mask)       # full recompute, as transformer.py:204
        last = logits[:, -1, :].contiguous()
        return ops.log_softmax(last, self.vocab_size), cache, attn

    def _inference_cached(self, preds, c):
        _no_train(self)
        pk = self._pack.get()
        if self.pos_emb.scale_learnable:
            raise NotImplementedError('decoder with learnable positional scale')
        c.begin_step(pk, preds)
        tok = preds[:, -1].contiguous()
        x = ops.embed_posenc(tok, pk['emb'], c.table, c.N, self.d_model, step_ptr=c.step_dev)
        x = self.decode_cached_bf16(pk, x, c.kc, c.vc, c.anc, c.step_dev, c.kvx, c.mem_len, c.beam, c.T)
        logits = ops.linear(x, pk['wout'], pk['bout'], EPI_BIAS, out_f32=True, n_out=self.ld_logits)
        c.step += 1
        attn = {'dec_block_%d' % i: {'slf_attn_weights': None, 'src_attn_weights': None} for i in range(len(self.blocks))}
        return ops.log_softmax(logits, self.vocab_size), c, attn
