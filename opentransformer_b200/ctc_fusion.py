"""LM shallow fusion in the CTC prefix beam search (DESIGN.md 4.19): ctcdecode's search with a neural LM as its scorer.

One frame is the search step (otb_ctc_prefix_beam_step: one CTA per utterance, the frame index from a device counter, the
slots in global memory) followed by one LM step over all B * beam rows; the frame runs T' times from the host without a
synchronisation, as a graphs.CapturedStep (the first frame eager, the others replays of its capture).  The LM state follows the slots: a row that kept its prefix carries its
source slot's LM row (and LSTM state), a row that extended runs the LM on its new token.

  * Recurrent LM: (h, c) per slot, gathered by source slot, then the embedding, the input GEMM, one otb_lstm_fwd step per
    layer, the head GEMM and otb_log_softmax.
  * Transformer LM: the K/V of each prefix node (node ids 1 + t * beam + s of DESIGN.md 4.7, 0 the BOS) are stored once
    per utterance, [blocks, B * (1 + T' * beam), d]; each row lists the cache rows of its prefix (anc, rewritten by the
    search step) and queries at its own position (otb_embed_posenc / otb_decode_self_attn with row_pos).
"""
import torch

from . import ops
from .graphs import CapturedStep

BOS = 1


class FusedLMRows:
    """The LM side of a fused search over N rows, shared by the CTC prefix beam search and the transducer's searches
    (DESIGN.md 4.19, 4.22).  The search step writes, per row: tok (i64) its newest token, ext (i32) 1 where the row took a
    new token, src (i32, optional) the row it continues; for the Transformer LM also anc / pos (the cache rows of the
    row's tokens from position 0, and the new token's position or -1).  follow() then makes lm_rows f32 [N, V] = log
    p_lm(. | <S/E>, row's tokens), and the recurrent LM's (h, c), follow the rows."""

    def _init_lm(self, lm, N, Lpos, cache_rows, bos_row, pos0, device):
        """Buffers for N rows; Transformer LM: cache_rows K/V rows per block, anc [N, Lpos], row n's <S/E> at cache row
        bos_row[n] and its first query position pos0[n] (-1: none)."""
        self.lm, self.N = lm, N
        i32 = dict(dtype=torch.int32, device=device)
        V = lm.vocab_size
        self.lm_rows = torch.zeros(N, V, dtype=torch.float32, device=device)
        self.lm_old = torch.zeros(N, V, dtype=torch.float32, device=device)
        self.src = torch.zeros(N, **i32)
        self.ext = torch.zeros(N, **i32)
        self.tok = torch.full((N,), BOS, dtype=torch.int64, device=device)
        self.anc = self.anc_tmp = self.pos = None
        if lm.model_type == 'transformer_lm':
            self.kc = torch.zeros(lm.num_blocks, cache_rows, lm.d_model, dtype=ops.BF16, device=device)
            self.vc = torch.zeros(lm.num_blocks, cache_rows, lm.d_model, dtype=ops.BF16, device=device)
            self.anc = torch.zeros(N, Lpos, **i32)
            self.anc_tmp = torch.zeros(N, Lpos, **i32)
            self.pos = torch.zeros(N, **i32)
            self.table = ops.sinusoid_table(Lpos + 1, lm.d_model, 0, device)
            self._pos0 = pos0.to(torch.int32)
            self._bos_row = bos_row.to(torch.int32)
        else:
            lm._check_device(device)
            shape = (lm.num_layers, N, lm.hidden_size)
            self.lm_h, self.lm_c = torch.zeros(shape, device=device), torch.zeros(shape, device=device)
            self.lm_h_old, self.lm_c_old = torch.zeros(shape, device=device), torch.zeros(shape, device=device)
            self._lstm_bar = torch.zeros(2, **i32)

    # ---- the kernels of one LM step over all rows ------------------------------------------------------------------
    def _lm_step(self):
        """LM rows of every row's newest token -> lm_rows (and, for the recurrent LM, the new (h, c) per layer)."""
        lm, N = self.lm, self.N
        pk = lm._pack.get()
        if self.anc is not None:
            x = ops.embed_posenc(self.tok, pk['emb'], self.table, N, lm.d_model, row_pos=self.pos)
            for l, (blk, p) in enumerate(zip(lm.blocks, pk['blocks'])):
                x = blk.run(x, p, N, 1, None, context=lambda qkv, l=l: ops.decode_self_attn(
                    qkv, self.kc[l], self.vc[l], self.anc, None, N, lm.n_heads, self.anc.shape[1], row_pos=self.pos))
            logits = ops.linear(x, pk['wout'], pk['bout'], ops.EPI_BIAS, out_f32=True, n_out=lm.ld_logits)
            ops.log_softmax(logits, lm.vocab_size, out=self.lm_rows)
            return None
        x = ops.embedding(self.tok, pk['emb'])
        new = []
        for k, p in enumerate(pk['layers']):
            gx = ops.linear(x, p['ih'].w, p['ih'].b, out_f32=True)
            x, h_n, c_n, _, _ = ops.lstm_fwd(gx, p['w_hh'], 1, N, self.lm_h_old[k], self.lm_c_old[k], barrier=self._lstm_bar)
            new.append((h_n, c_n))
        ops.log_softmax(lm._logits(x, pk), lm.vocab_size, out=self.lm_rows)
        return new

    def _take_state(self, new):
        """Rows that extended take the LM step's (h, c), the others their source slot's (already gathered)."""
        for k, (h_n, c_n) in enumerate(new):
            ops.ctc_lm_carry(self.lm_h[k], self.lm_h_old[k], ext=self.ext, a=h_n)
            ops.ctc_lm_carry(self.lm_c[k], self.lm_c_old[k], ext=self.ext, a=c_n)

    def follow(self, src):
        """After a search step: every row's LM rows and state from row src[n] (row n when src is None), advanced by the LM
        one token where ext[n]."""
        ops.ctc_lm_carry(self.lm_old, self.lm_rows, idx=src, ext=self.ext)           # kept rows: the source's LM row
        if self.anc is None:
            for k in range(self.lm.num_layers):
                ops.ctc_lm_carry(self.lm_h_old[k], self.lm_h[k], idx=src)
                ops.ctc_lm_carry(self.lm_c_old[k], self.lm_c[k], idx=src)
        new = self._lm_step()
        ops.ctc_lm_carry(self.lm_rows, self.lm_old, ext=self.ext)                     # ... put back over the LM's output
        if new is not None:
            self._take_state(new)

    def start_lm(self):
        """The LM on BOS for the empty sequence (the rows with a first position; every row for the recurrent LM)."""
        self.tok.fill_(BOS)
        self.ext.fill_(1)
        if self.anc is not None:
            self.anc[:, 0] = self._bos_row
            self.pos.copy_(self._pos0)
        else:
            self.lm_h_old.zero_()
            self.lm_c_old.zero_()
        new = self._lm_step()
        if new is not None:
            self._take_state(new)


class CTCFusedSearch(FusedLMRows):
    """The fused search for one (batch, beam, frames, top-K) geometry; every buffer is allocated here, before capture."""

    def __init__(self, lm, B, beam, T, K, device, lm_weight, beta, blank=0, use_graph=True):
        if lm.model_type == 'transformer_lm' and T > ops.DECODE_MAX_LEN:
            raise ValueError(f'CTC LM fusion: a prefix can be T\' = {T} tokens long and the Transformer LM\'s cached '
                             f'attention takes at most {ops.DECODE_MAX_LEN} positions')
        self.B, self.W, self.T, self.K = B, beam, T, K
        self.lm_weight, self.beta, self.blank = float(lm_weight), float(beta), blank
        N = B * beam
        i32 = dict(dtype=torch.int32, device=device)
        # Transformer LM cache rows: per utterance the BOS node and one node per (frame, slot); positions 0 .. T' - 1
        row = torch.arange(N, device=device)
        self._init_lm(lm, N, T, B * (1 + T * beam), (row // beam) * (1 + T * beam), torch.where(row % beam == 0, 0, -1),
                      device)
        self.top_lp = torch.zeros(B * T, K, dtype=torch.float32, device=device)
        self.top_id = torch.zeros(B * T, K, **i32)
        self.in_len = torch.zeros(B, **i32)
        self.slots = ops.ctc_prefix_beam_slots(B, device)
        self.ctl = torch.zeros(2, **i32)
        self.nodes = torch.zeros(B, 1 + T * beam, 2, **i32)
        self.ids = torch.zeros(B, beam, T, **i32)
        self.lengths = torch.zeros(B, beam, **i32)
        self.scores = torch.zeros(B, beam, dtype=torch.float32, device=device)
        # one frame, captured on the first and replayed; the graph bakes in the LM pack's addresses
        self.frame = CapturedStep(self._frame, self._packs, use_graph)

    @property
    def graph(self):
        """The captured frame (None until the first frame of the graph path)."""
        return self.frame.graph

    def _packs(self):
        return (self.lm._pack.get(),)

    def _frame(self):
        ops.ctc_prefix_beam_step(self.top_lp, self.top_id, self.B, self.T, self.in_len, self.W, self.blank, self.lm_rows,
                                 self.lm_weight, self.beta, self.slots, self.ctl, self.nodes, self.src, self.tok, self.ext,
                                 self.ids, self.lengths, self.scores, self.anc, self.anc_tmp, self.pos)
        self.follow(self.src)

    def _start(self):
        """Frame counter 0 and the LM on BOS for the empty prefix (slot 0 of every utterance)."""
        self.ctl.zero_()
        self.start_lm()

    def run(self, top_lp, top_id, in_len):
        """top_lp / top_id [B*T', K] of ctc_frame_topk, in_len i32 [B] -> (ids i64 [B, beam, T'] best first, lengths i32
        [B, beam], scores f32 [B, beam]: the fused totals log(p_b + p_nb))."""
        self.top_lp.copy_(top_lp)
        self.top_id.copy_(top_id)
        self.in_len.copy_(in_len)
        self._start()
        for _ in range(self.T):
            self.frame()
        return self.ids.long(), self.lengths.clone(), self.scores.clone()
