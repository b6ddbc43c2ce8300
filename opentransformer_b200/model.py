"""Model assembly with the reference's registries and checkpoint format.

Mirror of otrans/model/speech2text.py:14-87, otrans/model/__init__.py:6-9 and the three
string-keyed registries (frontend/__init__.py:8-12, encoder/__init__.py:10-13,
decoder/__init__.py:8-10).  A YAML `model:` section of the reference builds the CUDA model
unchanged; checkpoints written by the reference load through load_model() key for key.
"""
import torch
import torch.nn as nn

from . import ops
from .modules import ConformerEncoder, ConvFrontEnd, TransformerDecoder, TransformerEncoder, _lengths

BuildFrontEnd = {'conv': ConvFrontEnd}
BuildEncoder = {'transformer': TransformerEncoder, 'conformer': ConformerEncoder}
BuildDecoder = {'transformer': TransformerDecoder}


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

    def encode_bf16(self, inputs, mask):
        """frontend + encoder on the fused path -> (memory bf16 [B*T',D], lengths i32 [B], B, T')."""
        fe, enc = self.frontend, self.encoder
        B, T, _ = inputs.shape
        _, _, T2, _ = ops.conv_geometry(T, fe.input_size)
        lengths = _lengths(fe.output_mask(mask))
        if enc.fuse_abs_posenc():
            scale, table = enc.pos_emb.scale_and_table(T2, inputs.device)
            x, _ = fe.forward_bf16(inputs, scale, table)
        else:
            x, _ = fe.forward_bf16(inputs)
            x = enc.apply_posenc_bf16(x, B, T2)
        return enc.forward_bf16(x, B, T2, lengths), lengths, B, T2

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
        if self.training and torch.is_grad_enabled():
            from . import train
            loss, ctc = train.loss_with_grad(self, inputs['inputs'], inputs['mask'], truth, tlen)
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

    def _logits_padded(self, inputs, mask, targets_in):
        mem, lengths, B, T2 = self.encode_bf16(inputs, mask)
        return self.decoder.forward_bf16(targets_in, mem, lengths, B, targets_in.shape[1], T2)

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


End2EndModel = {'speech2text': SpeechToText}
