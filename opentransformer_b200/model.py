"""Model assembly with the reference's registries and checkpoint format.

Mirror of otrans/model/speech2text.py:14-87, otrans/model/__init__.py:6-9 and the three
string-keyed registries (frontend/__init__.py:8-12, encoder/__init__.py:10-13,
decoder/__init__.py:8-10).  A YAML `model:` section of the reference builds the CUDA model
unchanged; checkpoints written by the reference load through load_model() key for key.
"""
import torch
import torch.nn as nn

from . import ops
from . import train
from .lm import RecurrentLanguageModel, _LSTMParams
from .modules import (ConcatFeatureFrontEnd, ConcatWithLinearFrontEnd, ConformerEncoder, ConvFrontEnd, TransformerDecoder,
                      TransformerEncoder, _Packed, _lengths, _no_train, encoder_input_bf16)

BuildFrontEnd = {'concat': ConcatFeatureFrontEnd, 'concat-with-linear': ConcatWithLinearFrontEnd, 'conv': ConvFrontEnd}
BuildEncoder = {'transformer': TransformerEncoder, 'conformer': ConformerEncoder}
BuildDecoder = {'transformer': TransformerDecoder}


def ctc_align_logits(logits, lengths, B, T2, V, tokens, n_tokens, blank):
    """ops.ctc_align of a CTC head's logits f32 [B*T', ld] (first V columns valid) against tokens [B, Lmax] (n_tokens [B]
    of each row count), after the head's log-softmax."""
    lp = ops.log_softmax(logits, V).view(B, T2, V)
    n_tokens = n_tokens.to(device=logits.device, dtype=torch.int32).contiguous()
    return ops.ctc_align(lp, lengths, tokens, n_tokens, blank=blank)


def encoder_frames_to_input(spans, frame_shift=None, frontend=None):
    """Spans [start, end) in encoder frames (CTCModel.align, SpeechToText.align, CTCRecognizer.recognize_spans) -> spans in
    input (fbank) frames, [s start, s (end - 1) + w), where encoder frame t sees input frames [s t, s t + w): the front
    end's input_window() (s, w) -- (st1 st2, kt1 + (kt2 - 1) st1) for the conv front end, whose convolutions do not pad in
    time, and (stride, n) for the concat front ends.  Without a front end the shipped conv front end's window (4, 7) is
    used.  With frame_shift
    (seconds between input frames, e.g. 0.01) the result is in seconds, float64.  Entries of -1 (no span) stay -1."""
    s, w = frontend.input_window() if frontend is not None else (4, 7)
    out = torch.stack((s * spans[..., 0], s * (spans[..., 1] - 1) + w), dim=-1)
    if frame_shift is not None:
        out = out.double() * frame_shift
    return torch.where(spans < 0, -1, out)


class CTCAssistor(nn.Module):
    """model/ctc.py:12-66: the joint-CTC head, Linear(hidden, vocab) + nn.CTCLoss(blank = 0, zero_infinity).  Parameter
    holder (key `output_layer.*`, checkpoint section 'ctc'); compute is the wgmma GEMM + otb_ctc_loss."""

    def __init__(self, hidden_size, vocab_size, blank=0, lookahead_steps=-1):
        super().__init__()
        if lookahead_steps and lookahead_steps > 0:
            raise NotImplementedError('CTCAssistor lookahead convolution is not used by any shipped config')
        self.blank = blank
        self.vocab_size = vocab_size
        self.output_layer = nn.Linear(hidden_size, vocab_size)

    @property
    def ld_logits(self):
        return (self.vocab_size + 7) // 8 * 8

    def logits_bf16(self, mem_bf16):
        """memory bf16 [B*T', D] -> logits f32 [B*T', ld] (first V columns valid)."""
        w = self.output_layer.weight.detach().to(ops.BF16).contiguous()
        b = self.output_layer.bias.detach().float().contiguous()
        return ops.linear(mem_bf16, w, b, ops.EPI_BIAS, out_f32=True, n_out=self.ld_logits)

    def inference(self, memory, memory_mask):
        """model/ctc.py:54-66 -> (log_probs f32 [B,T,V], memory_length)."""
        B, T, D = memory.shape
        logits = self.logits_bf16(ops.scale_add_table(memory.contiguous().view(B * T, D).float()))
        lp = ops.log_softmax(logits, self.vocab_size)
        return lp.view(B, T, -1), _lengths(memory_mask.view(B, T))


class SpeechToText(nn.Module):
    def __init__(self, params):
        super().__init__()
        self.params = params
        self.frontend = BuildFrontEnd[params['frontend_type']](**params['frontend'])
        self.encoder = BuildEncoder[params['encoder_type']](**params['encoder'])
        self.decoder = BuildDecoder[params['decoder_type']](**params['decoder'])
        self.ctc_weight = params.get('ctc_weight', 0.0)
        if self.ctc_weight > 0.0:      # model/speech2text.py:30-36
            self.assistor = CTCAssistor(hidden_size=params['encoder_output_size'], vocab_size=params['decoder']['vocab_size'],
                                        lookahead_steps=params['lookahead_steps'] if 'lookahead_steps' in params else 0)
        self.smoothing = params.get('smoothing', 0.0)

    def encode_bf16(self, inputs, mask, attn_sink=None):
        """frontend + encoder on the fused path -> (memory bf16 [B*T',D], lengths i32 [B], B, T').  attn_sink (a list):
        each encoder block's attention weights f32 [B, H, T', T'] are appended to it."""
        fe, B = self.frontend, inputs.shape[0]
        _no_train(fe)
        x, lengths, T2, _ = encoder_input_bf16(fe, self.encoder, inputs, mask, fe._pack.get())
        return self.encoder.forward_bf16(x, B, T2, lengths, attn_sink), lengths, B, T2

    def forward_logits(self, inputs, mask, targets_in):
        """encoder + teacher-forced decoder (the forward half of speech2text.py:39-56) -> logits f32 [B,L,V]."""
        mem, lengths, B, T2 = self.encode_bf16(inputs, mask)
        L = targets_in.shape[1]
        logits = self.decoder.forward_bf16(targets_in, mem, lengths, B, L, T2)
        return logits.view(B, L, -1)[:, :, :self.decoder.vocab_size]

    def forward(self, inputs, targets):
        """SpeechToText.forward (model/speech2text.py:39-58) -> (loss, None).  In train mode with grad enabled the loss
        carries the hand-written backward (train.py): loss.backward() fills .grad of the fp32 parameters."""
        truth = targets['targets']
        tlen = targets.get('targets_length') if self.ctc_weight > 0.0 else None
        if self.ctc_weight > 0.0 and tlen is None:
            raise ValueError("joint CTC needs targets['targets_length'] (label count including <S/E>, data/loader.py:94)")
        # train() without gradients: a Conformer's BatchNorm must use the batch statistics and update its running buffers, as
        # the reference does; the inference path below would fold the running statistics instead
        if self.training and (torch.is_grad_enabled() or isinstance(self.encoder, ConformerEncoder)):
            run = train.loss_with_grad if torch.is_grad_enabled() else train.loss_train_mode
            loss, ctc = run(self, inputs['inputs'], inputs['mask'], truth, tlen), self._last_ctc_loss
            return loss, ({'CTCLoss': float(ctc)} if ctc is not None else None)
        mem, lengths, B, T2 = self.encode_bf16(inputs['inputs'], inputs['mask'])
        tin = truth[:, :-1].contiguous()
        logits_pad = self.decoder.forward_bf16(tin, mem, lengths, B, tin.shape[1], T2)
        loss, _ = ops.ls_cross_entropy(logits_pad, truth[:, 1:].contiguous(), self.decoder.vocab_size, self.smoothing)
        if self.ctc_weight > 0.0:      # speech2text.py:60-62
            lc, _, _ = ops.ctc_loss(self.assistor.logits_bf16(mem), B, T2, self.decoder.vocab_size, lengths,
                                    truth[:, 1:].contiguous(), tlen.to(torch.int32).to(mem.device).contiguous(), self.assistor.blank)
            return (1 - self.ctc_weight) * loss + self.ctc_weight * lc, {'CTCLoss': float(lc)}
        return loss, None

    def align(self, inputs, inputs_mask, targets, targets_length):
        """CTC forced alignment through the joint-CTC head, of the targets its loss scores: targets[:, 1:] with
        targets_length tokens (the reference's collate: <S/E> first, targets_length counts the labels after it, the closing
        <S/E> included).  -> ops.ctc_align's (labels i32 [B, T'], frame_scores f32 [B, T'], spans i32 [B, L, 2],
        path_score f32 [B]) on the device; spans are in encoder frames (encoder_frames_to_input converts them).  Runs the
        inference path, also in train().  A model without a CTC head (ctc_weight 0) raises ValueError."""
        if self.ctc_weight <= 0.0:
            raise ValueError('SpeechToText.align needs the joint-CTC head: this model has ctc_weight 0')
        with torch.no_grad():
            mem, lengths, B, T2 = self.encode_bf16(inputs, inputs_mask)
            return ctc_align_logits(self.assistor.logits_bf16(mem), lengths, B, T2, self.decoder.vocab_size, targets[:, 1:],
                                    targets_length, self.assistor.blank)

    train_pass = train.forward_backward
    mix_batch = train.mixspeech_halves

    def train_batch(self, inputs, mask, truth, truth_length=None):
        """FusedTrainer.step's arguments as train_pass takes them; it reads the label counts as int32."""
        return inputs, mask, truth, None if truth_length is None else truth_length.to(torch.int32)

    def check_fused_trainer(self):
        """Nothing is refused up front: the first pass builds the TrainPack, whose constructor checks the model."""

    def save_checkpoint(self, params, name):
        chk = {'params': params, 'frontend': self.frontend.state_dict(),
               'encoder': self.encoder.state_dict(), 'decoder': self.decoder.state_dict()}
        if self.ctc_weight > 0.0:
            chk['ctc'] = self.assistor.state_dict()
        torch.save(chk, name)

    def load_model(self, chkpt):
        self.frontend.load_state_dict(chkpt['frontend'])
        self.encoder.load_state_dict(chkpt['encoder'])
        self.decoder.load_state_dict(chkpt['decoder'])
        if self.ctc_weight > 0.0 and 'ctc' in chkpt:       # eval.py:43-45
            self.assistor.load_state_dict(chkpt['ctc'])

    def load_flat_state_dict(self, sd):
        """Load a flat {'frontend.x': ..} dict (test fixtures)."""
        for part in ('frontend', 'encoder', 'decoder'):
            sub = {k[len(part) + 1:]: v for k, v in sd.items() if k.startswith(part + '.')}
            getattr(self, part).load_state_dict(sub)

    def set_epoch(self, epoch):
        pass


class CTCModel(nn.Module):
    """model/ctc.py:69-131: front end + encoder + CTCAssistor, trained with nn.CTCLoss(blank 0, 'mean', zero_infinity)
    on truth[:, 1:-1] (no <S/E>) with targets_length - 1 labels.  Submodules `frontend`, `encoder`, `assistor`: the
    reference's state_dict keys and checkpoint sections.

    forward: train() with gradients -> one autograd node over the hand-written backward (train_pass);
    train() without gradients -> the training-mode forward (a Conformer's BatchNorm uses the batch statistics); eval() ->
    the fused inference path (encode_bf16, head GEMM, otb_ctc_loss)."""

    def __init__(self, params):
        super().__init__()
        self.params = params
        self.frontend = BuildFrontEnd[params['frontend_type']](**params['frontend'])
        self.encoder = BuildEncoder[params['encoder_type']](**params['encoder'])
        self.vocab_size = params['vocab_size']
        self.assistor = CTCAssistor(hidden_size=params['encoder_output_size'], vocab_size=self.vocab_size,
                                    lookahead_steps=params['lookahead_steps'] if 'lookahead_steps' in params else -1)

    encode_bf16 = SpeechToText.encode_bf16

    def logits_bf16(self, inputs, mask):
        """front end + encoder + CTC head -> (logits f32 [B*T', ld] (first V columns valid), lengths i32 [B], B, T')."""
        mem, lengths, B, T2 = self.encode_bf16(inputs, mask)
        return self.assistor.logits_bf16(mem), lengths, B, T2

    def forward(self, inputs, targets):
        """CTCModel.forward (model/ctc.py:83-96) -> (loss, None).  targets['targets_length'] (label count including <S/E>,
        data/loader.py:94) is required."""
        truth, tlen = targets['targets'], targets.get('targets_length')
        if tlen is None:
            raise ValueError("CTCModel needs targets['targets_length'] (label count including <S/E>, data/loader.py:94)")
        if self.training:
            run = train.loss_with_grad if torch.is_grad_enabled() else train.loss_train_mode
            return run(self, inputs['inputs'], inputs['mask'], truth, tlen), None
        logits, lengths, B, T2 = self.logits_bf16(inputs['inputs'], inputs['mask'])
        tl = (tlen.to(logits.device).to(torch.int32) - 1).contiguous()
        loss, _, _ = ops.ctc_loss(logits, B, T2, self.vocab_size, lengths, truth[:, 1:-1].contiguous(), tl, self.assistor.blank)
        return loss, None

    def inference(self, inputs, inputs_mask):
        """-> (log_probs f32 [B, T', V], lengths i32 [B]) of front end + encoder + head.  The reference's CTCModel.inference
        (model/ctc.py:98-103) skips the front end and unpacks the encoder's three return values into two, so it cannot run;
        this is what it evidently intends (DESIGN.md 6)."""
        logits, lengths, B, T2 = self.logits_bf16(inputs, inputs_mask)
        return ops.log_softmax(logits, self.vocab_size).view(B, T2, -1), lengths

    recognize = inference

    def align(self, inputs, inputs_mask, targets, targets_length):
        """CTC forced alignment of the transcripts, in forward's convention: targets[:, 1:-1] with targets_length - 1 tokens
        (the reference's collate, <S/E> at both ends and counted in targets_length).  One pass of the front end, encoder and
        head, then otb_ctc_align.  -> (labels i32 [B, T'] the token of each encoder frame, blank included, -1 past the
        utterance; frame_scores f32 [B, T'] its log-prob; spans i32 [B, L, 2] [start, end) of each token in encoder frames
        (encoder_frames_to_input converts them); path_score f32 [B] the best alignment's log-prob), on the device.  An
        utterance too short for its transcript gets -inf and -1.  Runs the inference path, also in train(): a Conformer's
        BatchNorm uses its running statistics and no dropout is applied."""
        with torch.no_grad():
            logits, lengths, B, T2 = self.logits_bf16(inputs, inputs_mask)
            return ctc_align_logits(logits, lengths, B, T2, self.vocab_size, targets[:, 1:-1], targets_length - 1,
                                    self.assistor.blank)

    train_pass = train.ctc_forward_backward
    mix_batch = train.mixspeech_halves
    check_fused_trainer = SpeechToText.check_fused_trainer

    def train_batch(self, inputs, mask, truth, truth_length=None):
        if truth_length is None:
            raise TypeError('FusedTrainer.step(inputs, mask, truth, truth_length) for a CTCModel: truth_length is required')
        return SpeechToText.train_batch(self, inputs, mask, truth, truth_length)

    def save_checkpoint(self, params, name):
        torch.save({'params': params, 'frontend': self.frontend.state_dict(), 'encoder': self.encoder.state_dict(),
                    'ctc': self.assistor.state_dict()}, name)

    def load_model(self, chkpt):
        """eval.py:36-57 for a CTC checkpoint: sections 'frontend' (when present), 'encoder' and 'ctc'."""
        if 'frontend' in chkpt:
            self.frontend.load_state_dict(chkpt['frontend'])
        self.encoder.load_state_dict(chkpt['encoder'])
        if 'ctc' in chkpt:
            self.assistor.load_state_dict(chkpt['ctc'])

    def set_epoch(self, epoch):
        pass


class PredictionNetwork(nn.Module):
    """The transducer's prediction network: embedding (V x hidden) and an LSTM stack with nn.LSTM's parameters
    (lm._LSTMParams: keys rnn.weight_ih_l0 ...), no output layer; dropout between layers in training.  Compute: the LSTM
    kernels of csrc/lstm.cu through train.lstm_stack_fwd / lstm_stack_bwd."""

    def __init__(self, vocab_size, hidden_size, num_layers=1, dropout=0.0):
        super().__init__()
        if hidden_size % 8:
            raise NotImplementedError(f'PredictionNetwork: the LSTM kernels need hidden_size a multiple of 8, got {hidden_size}')
        if not 0.0 <= float(dropout) < 1.0:
            raise ValueError(f'PredictionNetwork: dropout must be in [0, 1), got {dropout}')
        self.vocab_size, self.hidden_size, self.num_layers = vocab_size, hidden_size, num_layers
        self.dropout = float(dropout)
        self.embedding = nn.Embedding(vocab_size, hidden_size)
        self.rnn = _LSTMParams(hidden_size, hidden_size, num_layers)
        self._checked = None

    _check_device = RecurrentLanguageModel._check_device


class JointNetwork(nn.Module):
    """z = output_layer(tanh(enc_proj(h_t) + dec_proj(g_u))): enc_proj Linear(encoder d_model -> inner), dec_proj
    Linear(hidden -> inner, no bias), output_layer Linear(inner -> V).  Compute: otb_rnnt_joint between the projection
    GEMMs and the output layer's.

    prune_range S (an int >= 2, or None): pruned RNN-T training (DESIGN.md 4.22).  The simple joint simple_am_proj(h_t) +
    simple_lm_proj(g_u) (Linear(encoder d_model -> V), Linear(hidden -> V)) picks S label positions per frame, and the
    objective is simple_loss_scale * L_simple + L_pruned.  Recognition never reads the simple projections."""

    def __init__(self, encoder_size, hidden_size, inner_size, vocab_size, prune_range=None, simple_loss_scale=0.5):
        super().__init__()
        if inner_size % 8:
            raise NotImplementedError(f'JointNetwork: the joint kernels need inner_size a multiple of 8, got {inner_size}')
        if prune_range is not None and (isinstance(prune_range, bool) or not isinstance(prune_range, int) or prune_range < 2):
            raise ValueError(f'JointNetwork: prune_range must be an int >= 2 or None, got {prune_range!r}')
        if isinstance(simple_loss_scale, bool) or not isinstance(simple_loss_scale, (int, float)) or not simple_loss_scale >= 0:
            raise ValueError(f'JointNetwork: simple_loss_scale must be a number >= 0, got {simple_loss_scale!r}')
        self.inner_size, self.vocab_size = inner_size, vocab_size
        self.prune_range, self.simple_loss_scale = prune_range, float(simple_loss_scale)
        self.enc_proj = nn.Linear(encoder_size, inner_size)
        self.dec_proj = nn.Linear(hidden_size, inner_size, bias=False)
        self.output_layer = nn.Linear(inner_size, vocab_size)
        if prune_range is not None:
            self.simple_am_proj = nn.Linear(encoder_size, vocab_size)
            self.simple_lm_proj = nn.Linear(hidden_size, vocab_size)

    @property
    def ld_logits(self):
        return (self.vocab_size + 7) // 8 * 8


class TransducerModel(nn.Module):
    """RNN-T (DESIGN.md 4.22): front end + encoder as for SpeechToText, a PredictionNetwork (`decoder`, over [BLK, y_1 ..
    y_U]) and a JointNetwork (`joint`), trained with the transducer loss -- the negative log-likelihood of the transcript
    summed over all alignments of the [T', U + 1] lattice, averaged over the batch (torchaudio.functional.rnnt_loss with
    reduction 'mean') -- on truth[:, 1:-1] with targets_length - 1 labels, blank BLK = 0.  Checkpoint sections
    'frontend', 'encoder', 'decoder', 'joint' (what eval.py loads).

    forward: train() with gradients -> one autograd node over the hand-written backward (train_pass); train() without
    gradients -> the training-mode forward; eval() -> the fused inference pass.  Greedy recognition: TransducerRecognizer."""

    def __init__(self, params):
        super().__init__()
        self.params = params
        if params.get('decoder_type', 'rnn') != 'rnn':
            raise NotImplementedError(f"TransducerModel: decoder_type {params['decoder_type']!r}; the prediction network is an "
                                      "LSTM stack ('rnn')")
        self.frontend = BuildFrontEnd[params['frontend_type']](**params['frontend'])
        self.encoder = BuildEncoder[params['encoder_type']](**params['encoder'])
        self.decoder = PredictionNetwork(**params['decoder'])
        self.vocab_size = self.decoder.vocab_size
        jp = params['joint']
        self.joint = JointNetwork(self.encoder.d_model, self.decoder.hidden_size, jp['inner_size'], self.vocab_size,
                                  jp.get('prune_range'), jp.get('simple_loss_scale', 0.5))
        self.blank = 0
        # the inference pack (recognition and the eval-mode loss); the simple projections, which only the pruned loss
        # reads, are cast separately
        self._pack = _Packed(self, lambda: train.transducer_operands(self, train.LayerPack(self), simple=False))
        self._simple_pack = _Packed(self, lambda: train.simple_operands(self, train.LayerPack(self)))

    encode_bf16 = SpeechToText.encode_bf16

    def forward(self, inputs, targets):
        """-> (loss, None).  targets['targets_length'] (label count including <S/E>, data/loader.py:94) is required."""
        truth, tlen = targets['targets'], targets.get('targets_length')
        if tlen is None:
            raise ValueError("TransducerModel needs targets['targets_length'] (label count including <S/E>, data/loader.py:94)")
        if self.training:
            run = train.loss_with_grad if torch.is_grad_enabled() else train.loss_train_mode
            return run(self, inputs['inputs'], inputs['mask'], truth, tlen), None
        with torch.no_grad():
            mem, lengths, B, T2 = self.encode_bf16(inputs['inputs'], inputs['mask'])
            op = self._pack.get()
            if self.joint.prune_range is not None:
                op = dict(op, simple=self._simple_pack.get())
            loss, _ = train.transducer_head(self, op, mem, B, T2, lengths, truth, tlen)
        return loss, None

    train_pass = train.transducer_forward_backward
    mix_batch = train.mixspeech_halves
    check_fused_trainer = SpeechToText.check_fused_trainer

    def train_batch(self, inputs, mask, truth, truth_length=None):
        if truth_length is None:
            raise TypeError('FusedTrainer.step(inputs, mask, truth, truth_length) for a TransducerModel: truth_length is required')
        return SpeechToText.train_batch(self, inputs, mask, truth, truth_length)

    def save_checkpoint(self, params, name):
        torch.save({'params': params, 'frontend': self.frontend.state_dict(), 'encoder': self.encoder.state_dict(),
                    'decoder': self.decoder.state_dict(), 'joint': self.joint.state_dict()}, name)

    def load_model(self, chkpt):
        """eval.py:36-49 for a transducer checkpoint: sections 'frontend' (when present), 'encoder', 'decoder' and 'joint'."""
        if 'frontend' in chkpt:
            self.frontend.load_state_dict(chkpt['frontend'])
        self.encoder.load_state_dict(chkpt['encoder'])
        self.decoder.load_state_dict(chkpt['decoder'])
        self.joint.load_state_dict(chkpt['joint'])

    def set_epoch(self, epoch):
        pass


End2EndModel = {'ctc': CTCModel, 'speech2text': SpeechToText, 'transducer': TransducerModel}
