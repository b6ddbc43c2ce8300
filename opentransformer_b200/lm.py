"""Language models for shallow fusion and training on the CUDA path: the two model types of otrans/model/lm.py.

TransformerLanguageModel mirrors lm.py:93-171: embedding + sinusoidal positions + ``num_blocks`` post-norm
TransformerEncoderLayers (GLU FFN) under a causal mask + tied output projection, on the same sm_90a kernels as the acoustic
encoder (causal flag on the attention kernel).  ``lm.train(); loss, _ = lm(inputs, targets); loss.backward()`` fills
``.grad`` of every parameter through the speech encoder layer's hand-written training forward and backward (train.py) with
the causal mask.  Training needs 64-wide heads, the width of the attention backward.

RecurrentLanguageModel mirrors lm.py:31-90 (rnnlm.yaml): embedding -> ``num_layers`` nn.LSTM layers (dropout between them
in training) -> output projection, optionally tied to the embedding.  Each layer is one GEMM for the input projection of all
positions and the persistent recurrence kernels of csrc/lstm.cu; ``lm.train(); loss, _ = lm(inputs, targets);
loss.backward()`` fills ``.grad`` of every parameter through a hand-written backward through time.

Both plug into training by train.py's contract (``train_pass`` / ``check_fused_trainer``, and ``train_batch`` where
``train.FusedTrainer`` takes the model: the Transformer LM, whose TransformerScheduler is the one it keeps on the device; the
recurrent LM's step-linear scheduler is not, so it is refused).

Both keep the reference's constructor (``params`` dict of the YAML ``model:`` section), ``state_dict`` keys and ``predict``
signature.  The recogniser adds ``lm_weight * log_probs`` inside the fused log-softmax/top-k kernel
(recognize/speech2text.py:102-105 -> otb_logsoftmax_topk).
"""
import math

import torch
import torch.nn as nn

from . import ops
from . import train
from .modules import BF16, PositionalEncoding, SelfAttnCache, TransformerEncoderLayer, _Packed, _b, _no_train, _w


class LMCache(SelfAttnCache):
    """The incremental state of the Transformer LM that the reference stubbed out (recognize/speech2text.py:142-143 leaves
    the reorder of cache['lm'] commented out), as the `cache` of ``TransformerLanguageModel.predict(targets, True, cache)``:
    the self-attention K/V of every position each block has seen [block, position, row, d_model] (SelfAttnCache).  One
    call consumes one new token per row; ``reorder(parent_rows)`` follows beam pruning without moving K/V rows.

    Build it with ``TransformerLanguageModel.init_cache``."""

    def __init__(self, lm, n_rows, max_len, anc=None, step_ptr=None):
        if n_rows < 1:
            raise ValueError(f'LMCache: n_rows must be >= 1, got {n_rows}')
        if not 1 <= max_len <= ops.DECODE_MAX_LEN:
            raise ValueError(f'LMCache: max_len must be in [1, {ops.DECODE_MAX_LEN}], got {max_len}')
        super().__init__('LM', lm._pack.get(), lm.num_blocks, n_rows, lm.d_model, max_len, lm.embedding.weight.device, anc,
                         step_ptr)


class TransformerLanguageModel(nn.Module):
    def __init__(self, params):
        super().__init__()
        self.params = params
        self.model_type = 'transformer_lm'
        self.normalize_before = False
        self.smoothing = params.get('smoothing', 0.0)
        self.vocab_size = params['vocab_size']
        self.num_blocks = params['num_blocks']
        self.d_model = params['d_model']
        self.n_heads = params['n_heads']
        self.embedding = nn.Embedding(self.vocab_size, self.d_model)
        self.pos_embedding = PositionalEncoding(self.d_model, 0.0)
        self.blocks = nn.ModuleList([
            TransformerEncoderLayer(params['n_heads'], self.d_model, params['d_ff'], slf_attn_dropout=0.0,
                                    ffn_dropout=0.0, residual_dropout=params.get('residual_dropout', 0.0),
                                    normalize_before=False, concat_after=False, activation='glu')
            for _ in range(self.num_blocks)])
        self.output_project = nn.Linear(self.d_model, self.vocab_size)
        if params.get('share_embedding', False):
            self.output_project.weight = self.embedding.weight
        self._pack = _Packed(self, self._build_pack)

    def _build_pack(self):
        emb = self.embedding.weight.detach().to(BF16).contiguous()
        tied = self.output_project.weight is self.embedding.weight
        return {'emb': emb, 'wout': emb if tied else _w(self.output_project), 'bout': _b(self.output_project),
                'blocks': [b.pack() for b in self.blocks]}

    @property
    def ld_logits(self):
        return (self.vocab_size + 7) // 8 * 8

    def logits_bf16(self, targets):
        """targets i64 [N,L] -> logits f32 [N*L, ld_logits] (full prefix, as the reference recomputes it)."""
        _no_train(self)
        pk = self._pack.get()
        N, L = targets.shape
        scale, table = self.pos_embedding.scale_and_table(L, targets.device)
        x = ops.embed_posenc(targets.contiguous(), pk['emb'], table, N * L, self.d_model, period=L)
        for blk, p in zip(self.blocks, pk['blocks']):
            x = blk.run(x, p, N, L, None, causal=True)
        return ops.linear(x, pk['wout'], pk['bout'], ops.EPI_BIAS, out_f32=True, n_out=self.ld_logits)

    def init_cache(self, n_rows, max_len):
        """KV cache for ``predict(targets, True, cache)`` over n_rows sequences of at most max_len positions (LMCache)."""
        _no_train(self)
        return LMCache(self, n_rows, max_len)

    def cached_log_probs(self, pk, tok, c, out=None):
        """The newest position of every row through the blocks against the KV cache c (LMCache): tok i64 [N] at the position
        c.step_dev names -> log-probs f32 [N, V].  Each block's K/V of that position are written into the cache; earlier
        positions are read through c.anc."""
        N, H = c.N, self.n_heads
        x = ops.embed_posenc(tok, pk['emb'], c.table, N, self.d_model, step_ptr=c.step_dev)
        for l, (blk, p) in enumerate(zip(self.blocks, pk['blocks'])):
            x = blk.run(x, p, N, 1, None, context=lambda qkv, l=l: ops.decode_self_attn(qkv, c.kc[l], c.vc[l], c.anc,
                                                                                        c.step_dev, N, H, c.Lmax))
        logits = ops.linear(x, pk['wout'], pk['bout'], ops.EPI_BIAS, out_f32=True, n_out=self.ld_logits)
        return ops.log_softmax(logits, self.vocab_size, out=out)

    def predict(self, targets, last_frame=True, cache=None):
        """model/lm.py:143-163: log-probs [N,1,V] of the last position, or [N,L,V] of all positions.

        cache None (the reference's only mode): the whole prefix is recomputed.  cache = LMCache (``init_cache``): targets
        is [N, cache.step + 1] and only targets[:, -1] runs through the blocks, at position cache.step, against the cached
        K/V of the earlier positions; the caller reorders the cache after beam pruning
        (SpeechToTextRecognizer.decode_step does)."""
        if cache is not None:
            if not isinstance(cache, LMCache):
                raise TypeError(f'predict: cache must be an LMCache (init_cache) or None, got {type(cache).__name__}')
            if not last_frame:
                raise ValueError('predict with an LMCache returns the newest position only: last_frame must be True')
            _no_train(self)
            pk = self._pack.get()
            cache.begin_step(pk, targets)
            with torch.no_grad():
                lp = self.cached_log_probs(pk, targets[:, -1].contiguous(), cache)
            cache.step += 1
            return lp.unsqueeze(1)
        N, L = targets.shape
        with torch.no_grad():
            logits = self.logits_bf16(targets).view(N, L, -1)
            if last_frame:
                last = logits[:, -1, :].contiguous()
                return ops.log_softmax(last, self.vocab_size).unsqueeze(1)
            flat = logits.reshape(N * L, -1)
            return ops.log_softmax(flat, self.vocab_size).view(N, L, self.vocab_size)

    def forward(self, inputs, targets):
        """model/lm.py:126-141: label-smoothed CE of the next-token prediction, PAD ignored -> (loss, None).  In training
        mode with gradients enabled, loss.backward() fills .grad of every parameter; in training mode without gradients
        the training forward (residual dropout on) runs alone."""
        if self.training:
            self.check_trainable()          # before the dropout seed is drawn: no device work ahead of a refusal
            run = train.loss_with_grad if torch.is_grad_enabled() else train.loss_train_mode
            return run(self, inputs['inputs'], targets['targets']), None
        with torch.no_grad():
            logits = self.logits_bf16(inputs['inputs'])
            loss, _ = ops.ls_cross_entropy(logits, targets['targets'].contiguous(), self.vocab_size, self.smoothing)
        return loss, None

    def check_trainable(self):
        """Refuse, before any device work, what the training path does not cover -> the residual_dropout rate of every block."""
        train.check_heads('language model', self.d_model, self.blocks)
        return train.check_blocks(self.blocks)

    check_fused_trainer = check_trainable

    def train_batch(self, inputs, targets):
        return inputs, targets

    def train_pass(self, inputs, targets, want_grads=True, grad_sink=None, grad_scale=1.0, bf16_of=None, drop_seed=None):
        """Training-mode forward (and hand-written backward) of model/lm.py:126-141, by train.py's contract: inputs / targets
        i64 [N, L] (targets PAD-padded) -> (loss 0-d f32, {parameter name -> fp32 gradient} or None).

        The mask is get_seq_mask (lm.py:14-18): the causal tril only, no key-padding mask.  Padding sits at the end of a row,
        so a padded position sees earlier padded positions but no scored position ever reads one, and PAD targets are left out
        of the loss: causal attention without kv_len gives the reference's loss and gradients exactly."""
        rates = self.check_trainable()
        train.need_drop_seed(drop_seed, rates)
        pk = train.LayerPack(self, bf16_of)
        blocks = [pk.enc_layer(b) for b in self.blocks]
        emb = pk.w(self.embedding.weight)
        tied = self.output_project.weight is self.embedding.weight
        wout = emb if tied else pk.w(self.output_project.weight)
        bout = self.output_project.bias.detach().float().contiguous()
        tok = inputs.contiguous()
        N, L = tok.shape
        d, H, V = self.d_model, self.blocks[0].n_heads, self.vocab_size
        _, table = self.pos_embedding.scale_and_table(L, tok.device)
        x = ops.embed_posenc(tok, emb, table, N * L, d, period=L)                       # x * sqrt(d) + PE, dropout 0
        drops = [(r, drop_seed, TLM_SITE + 2 * i) for i, r in enumerate(rates)]
        tape = []
        for p, drop in zip(blocks, drops):
            x, t = train.enc_layer_fwd(p, x, False, N, H, L, None, drop, causal=True)
            tape.append(t)
        logits = train.head_fwd(x, wout, bout, self.ld_logits)
        if not want_grads:
            loss, _ = ops.ls_cross_entropy(logits, targets.contiguous(), V, self.smoothing)
            return loss, None
        loss, dlogits = ops.ls_cross_entropy_train(logits, targets.contiguous(), V, self.smoothing)
        if grad_scale != 1.0:
            dlogits = ops.scale_add_table(dlogits, grad_scale)                           # loss / accum_steps (trainer.py:216)
        g = train.Grads(grad_sink)
        dx = train.head_bwd(dlogits, x, wout, g, 'embedding.weight' if tied else 'output_project.weight', 'output_project.bias')
        for i in reversed(range(len(blocks))):
            dx = train.enc_layer_bwd(blocks[i], tape[i], dx, False, g, N, H, L, None, drops[i], causal=True)
        train.embedding_bwd(tok, dx, emb, math.sqrt(d), g, 'embedding.weight')
        return loss, g

    def save_checkpoint(self, params, name):
        torch.save({'params': params, 'model': self.state_dict()}, name)


# dropout sites of the Transformer LM's block i: TLM_SITE + 2 i + {0: after self-attention, 1: after the feed-forward}
# (train.ENC_SITE / DEC_SITE for the speech model, RNNLM_SITE for the recurrent LM)
TLM_SITE = 3000

transformer_forward_backward = TransformerLanguageModel.train_pass      # the pass as a function of the model

RNNLM_SITE = 2000      # dropout site of the output of LSTM layer k: RNNLM_SITE + k (train.ENC_SITE / DEC_SITE for the speech model)


class _LSTMParams(nn.Module):
    """Parameter holder with nn.LSTM's names, shapes and initialisation (weight_ih_l{k} [4H, I], weight_hh_l{k} [4H, H],
    bias_ih_l{k}, bias_hh_l{k} [4H]; gates ordered i, f, g, o).  Its forward is never run: the layers run on csrc/lstm.cu."""

    def __init__(self, input_size, hidden_size, num_layers):
        super().__init__()
        self.num_layers, self.hidden_size = num_layers, hidden_size
        for k in range(num_layers):
            i = input_size if k == 0 else hidden_size
            for name, shape in (('weight_ih', (4 * hidden_size, i)), ('weight_hh', (4 * hidden_size, hidden_size)),
                                ('bias_ih', (4 * hidden_size,)), ('bias_hh', (4 * hidden_size,))):
                self.register_parameter(f'{name}_l{k}', nn.Parameter(torch.empty(shape)))
        bound = 1.0 / math.sqrt(hidden_size)
        for p in self.parameters():
            nn.init.uniform_(p, -bound, bound)


class RecurrentLanguageModel(nn.Module):
    def __init__(self, params):
        super().__init__()
        self.params = params
        self.model_type = 'recurrent_lm'
        self.vocab_size = params['vocab_size']
        self.share_embedding = params['share_embedding']
        self.smoothing = params['smoothing']
        self.num_layers = params['num_layers']
        self.hidden_size = params['hidden_size']
        self.dropout = float(params['dropout'])          # residual_dropout is accepted and unused, as in the reference
        if self.hidden_size % 8:
            raise NotImplementedError(f'RecurrentLanguageModel: the LSTM kernels need hidden_size a multiple of 8, got {self.hidden_size}')
        self.embedding = nn.Embedding(self.vocab_size, self.hidden_size)
        self.rnn = _LSTMParams(self.hidden_size, self.hidden_size, self.num_layers)
        self.output_project = nn.Linear(self.hidden_size, self.vocab_size)
        if self.share_embedding:
            self.output_project.weight = self.embedding.weight
        self._pack = _Packed(self, self._build_pack)
        self._checked = None

    @property
    def ld_logits(self):
        return (self.vocab_size + 7) // 8 * 8

    def _build_pack(self):
        emb = self.embedding.weight.detach().to(BF16).contiguous()
        tied = self.output_project.weight is self.embedding.weight
        layers = train.lstm_layers(self.rnn, lambda p: p.detach().to(BF16).contiguous(), 'rnn.')
        return {'emb': emb, 'wout': emb if tied else _w(self.output_project), 'bout': _b(self.output_project), 'layers': layers}

    def _check_device(self, device):
        """The recurrence kernels keep a slice of W_hh per CTA in shared memory: refuse a hidden size whose slice does not
        fit this device."""
        if self._checked != device:
            prop = torch.cuda.get_device_properties(device)
            ops.lstm_config(self.hidden_size, prop.multi_processor_count, prop.shared_memory_per_block_optin)
            self._checked = device

    def _run(self, tok, pk, hidden=None, drop_seed=None, record=False, barrier=None):
        """tok i64 [L, N] (time-major) -> (output of the top layer bf16 [L*N, H], h_n, c_n f32 [layers, N, H], tape).
        hidden: (h0, c0) f32 [layers, N, H] or None; drop_seed: the dropout seed (training), else no dropout; record: keep
        what the backward reads (per layer: input, gates, c_t, output); barrier: see ops.lstm_fwd."""
        self._check_device(tok.device)
        L, N = tok.shape
        x = ops.embedding(tok.reshape(-1), pk['emb'])
        return train.lstm_stack_fwd(x, pk['layers'], L, N, self.dropout, drop_seed, RNNLM_SITE, hidden, record, barrier)

    def _logits(self, x, pk):
        return train.head_fwd(x, pk['wout'], pk['bout'], self.ld_logits)

    def init_hidden_states(self, batch_size, device):
        return torch.zeros([self.num_layers, batch_size, self.hidden_size]).to(device)

    def predict(self, pred, hidden=None):
        """model/lm.py:80-86: pred i64 [N, L], hidden (h, c) f32 [layers, N, H] or None (zero state)
        -> (log-probs f32 [N, L, V], (h_n, c_n) f32 [layers, N, H])."""
        N, L = pred.shape
        with torch.no_grad():
            pk = self._pack.get()
            x, h_n, c_n, _ = self._run(pred.t().contiguous(), pk, hidden)
            logp = ops.log_softmax(self._logits(x, pk), self.vocab_size)
            return logp.view(L, N, self.vocab_size).transpose(0, 1).contiguous(), (h_n, c_n)

    def forward(self, inputs, targets):
        """model/lm.py:62-73: label-smoothed CE of the next-token logits, PAD ignored -> (loss, None).  In training mode with
        gradients enabled, loss.backward() fills .grad of every parameter."""
        if self.training:
            run = train.loss_with_grad if torch.is_grad_enabled() else train.loss_train_mode
            return run(self, inputs['inputs'], targets['targets']), None
        with torch.no_grad():
            pk = self._pack.get()
            x, _, _, _ = self._run(inputs['inputs'].t().contiguous(), pk)
            loss, _ = ops.ls_cross_entropy(self._logits(x, pk), targets['targets'].t().contiguous(), self.vocab_size, self.smoothing)
        return loss, None

    def check_fused_trainer(self):
        raise NotImplementedError('FusedTrainer: the recurrent LM trains with a step-linear scheduler that is not on the '
                                  'device; train it through loss.backward() and a torch optimizer')

    def train_pass(self, inputs, targets, want_grads=True, drop_seed=None):
        """Training-mode forward and hand-written backward, by train.py's contract (FusedTrainer does not take this model, so
        without its grad_sink / grad_scale / bf16_of): inputs / targets i64 [N, L] (targets PAD-padded) -> (loss 0-d f32,
        {parameter name -> fp32 gradient} or None).  drop_seed: int32 device tensor [1], needed when dropout > 0
        (applied to the output of every layer but the last)."""
        train.need_drop_seed(drop_seed, [self.dropout] * (self.num_layers - 1))
        pk = self._pack.get()
        tok = inputs.t().contiguous()
        L, N = tok.shape
        V = self.vocab_size
        x, _, _, tape = self._run(tok, pk, drop_seed=drop_seed, record=want_grads)
        if not want_grads:
            loss, _ = ops.ls_cross_entropy(self._logits(x, pk), targets.t().contiguous(), V, self.smoothing)
            return loss, None
        loss, dlogits = ops.ls_cross_entropy_train(self._logits(x, pk), targets.t().contiguous(), V, self.smoothing)
        g = train.Grads()
        tied = self.output_project.weight is self.embedding.weight
        dy = train.head_bwd(dlogits, x, pk['wout'], g, 'embedding.weight' if tied else 'output_project.weight', 'output_project.bias')
        dy = train.lstm_stack_bwd(dy, tape, pk['layers'], L, N, g, self.dropout, drop_seed, RNNLM_SITE)
        train.embedding_bwd(tok, dy, pk['emb'], 1.0, g, 'embedding.weight')
        return loss, g

    def save_checkpoint(self, params, name):
        torch.save({'params': params, 'model': self.state_dict()}, name)


LanguageModel = {'transformer_lm': TransformerLanguageModel, 'rnn_lm': RecurrentLanguageModel}
