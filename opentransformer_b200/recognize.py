"""Batched beam-search recogniser on the CUDA hot path.

Mirror of otrans/recognize/speech2text.py (SpeechToTextRecognizer) and the bits of
otrans/recognize/base.py it needs.  Same constructor, same ``recognize`` / ``encode`` / ``decode`` /
``decode_step`` seams and return types.  What changes underneath:

  * encode: conv front end + encoder run as hand-written sm_90a kernels (bf16 tensor cores);
  * decode: the reference re-runs the whole decoder over the whole prefix -- and the cross-attention
    K/V projection of the beam-tiled memory -- at every step (decoder/transformer.py:204,
    attention.py:129).  Here cross K/V are projected ONCE per utterance (shared by the beams), self-attention
    K/V live in a per-hypothesis cache addressed through a 4-byte ancestry table, and one step is
    a fixed sequence of kernels captured in a CUDA graph and replayed;
  * beam step: one kernel per step (top-k, finished masking, pruning, back-pointers), no host sync
    inside the loop except a 4-byte "all ended" poll every few steps;
  * joint CTC/attention decoding (ctc_weight > 0, which the reference stores and never reads): the CTC prefix score of the
    joint-CTC head re-ranks each hypothesis' best candidates inside the step (csrc/ctc_prefix.cu, DESIGN.md 4.9);
  * n-best rescoring (apply_rescoring / apply_lm_rescoring / rescore_weight, which the reference parses and never passes
    on): a teacher-forced second pass of the attention decoder or an LM re-ranks the first pass's n-best
    (csrc/rescore.cu, DESIGN.md 4.10);
  * CTC rescoring (apply_ctc_rescoring): the joint-CTC head's full-sequence log-likelihood re-ranks the attention search's
    n-best (csrc/ctc_score.cu, DESIGN.md 4.18);
  * CTC LM fusion (CTCRecognizer(lm_fusion=True)): the neural LM is ctcdecode's scorer inside the CTC prefix beam search
    (ctc_fusion.py, DESIGN.md 4.19).
"""
import torch

from . import ops
from . import train
from .ctc_fusion import CTCFusedSearch, FusedLMRows
from .graphs import CapturedStep, lru_get, read_device
from .lm import LMCache
from .model import ctc_align_logits
from .modules import encoder_attn_weights

PAD, BOS, EOS = 0, 1, 1   # otrans/data/__init__.py:7-10


class Recognizer:
    """otrans/recognize/base.py:5-24,91-119 (model holder + id -> string translation)."""

    def __init__(self, model, idx2unit=None, lm=None, lm_weight=None, ngpu=1):
        self.ngpu = ngpu
        self.model = model
        self.model.eval()
        if self.ngpu > 0:
            self.model.cuda()
        self.lm = lm
        if self.lm is not None:
            self.lm.eval()
            if self.ngpu > 0:
                self.lm.cuda()
        self.idx2unit = idx2unit
        self.lm_weight = lm_weight

    def lm_decode(self, preds, hidden=None):
        """recognize/base.py:26-37: the Transformer LM re-reads the whole prefix, the RNN LM reads the newest token from
        `hidden`."""
        if self.lm.model_type == 'transformer_lm':
            return self.lm.predict(preds, last_frame=True), hidden
        return self.lm.predict(preds[:, -1:], hidden)

    def translate(self, seqs):
        results = []
        for seq in seqs:
            pred = []
            for i in seq:
                if int(i) == EOS:
                    break
                if int(i) == PAD:
                    continue
                pred.append(self.idx2unit[int(i)])
            results.append(' '.join(pred))
        return results

    def nbest_translate(self, nbest_preds):
        assert nbest_preds.dim() == 3
        if self.idx2unit is None:          # ids requested (tests / benchmarks): keep the tensor
            return nbest_preds
        rows = nbest_preds.cpu().tolist()
        results = []
        for per_utt in rows:
            nbest_list = []
            for seq in per_utt:
                pred = []
                for token in seq:
                    if token == EOS:
                        break
                    pred.append(self.idx2unit[token])
                nbest_list.append(' '.join(pred))
            results.append(nbest_list)
        return results


def lm_log_probs(lm, preds):
    """The LM term of one shallow-fusion step (speech2text.py:102-105 through base.py:26-37): log-probs f32 [N, V] of the
    token after each prefix preds i64 [N, l].  The RNN LM gets the newest token and NO carried state: the reference hands
    lm_decode cache['lm'] = None at every step (speech2text.py:41,103) and never stores the hidden state it returns."""
    if lm.model_type == 'transformer_lm':
        return lm.predict(preds, last_frame=True).squeeze(1).contiguous()
    return lm.predict(preds[:, -1:], None)[0].squeeze(1).contiguous()


def lm_token_logprob(lm, inputs, targets):
    """Token log-probs f32 [N, Lp] of targets i32 [N, Lp] (-1 after a sequence's end: 0 there) under the LM teacher-forced
    on inputs i64 [N, Lp]: the Transformer LM's full-sequence logits, the recurrent LM's from a zero state.  Neither lets a
    position see later ones, so the padding after a sequence's end needs no mask."""
    N, Lp = targets.shape
    if lm.model_type == 'transformer_lm':
        return ops.token_logprob(lm.logits_bf16(inputs), lm.vocab_size, targets.reshape(-1)).view(N, Lp)
    pk = lm._pack.get()
    x, _, _, _ = lm._run(inputs.t().contiguous(), pk)                      # time-major rows
    return ops.token_logprob(lm._logits(x, pk), lm.vocab_size, targets.t().reshape(-1)).view(Lp, N).t()


def second_pass_rows(ids, lengths=None):
    """The sequences a second pass scores, from first-pass ids [B, K, W] (DESIGN.md 4.10): hypothesis y is its row cut at
    the first <S/E> (and at `lengths` [B, K] when given: the CTC n-best's rows end in 0s), and the scored sequence is
    y <S/E>.  -> (inputs i64 [B*K, Lp] = BOS y PAD..., targets i32 [B, K, Lp] = y <S/E> -1..., n i32 [B, K] the length
    of y, Lp = max n + 1).  Reading Lp is the one host synchronisation."""
    B, K, W = ids.shape
    dev = ids.device
    ext = torch.cat((ids.long(), torch.full((B, K, 1), EOS, dtype=torch.int64, device=dev)), dim=2)
    if lengths is not None:
        ext = torch.where(torch.arange(W + 1, device=dev) >= lengths[..., None], EOS, ext)
    n = (ext == EOS).int().argmax(dim=2)                                      # the first <S/E>
    Lp = int(n.max()) + 1
    pos = torch.arange(Lp, device=dev)
    targets = torch.where(pos < n[..., None], ext[:, :, :Lp], torch.where(pos == n[..., None], EOS, -1)).int()
    inputs = torch.cat((torch.full((B, K, 1), BOS, dtype=torch.int64, device=dev), targets[:, :, :-1].clamp_min(PAD).long()), 2)
    return inputs.view(B * K, Lp), targets, n.int(), Lp


def error_counts(ids, lengths, truth, truth_length):
    """eval.py's token error counts of one batch, on the device and without a host synchronisation: ids [B, K, W] a
    recognizer's n-best as recognize_ids returns it, each row cut at its first <S/E> (and at lengths i32 [B, K] when given:
    the CTC recognizers' rows), scored by otb_edit_distance against truth[b, 1 : truth_length[b]] (truth i64 [B, L + 1],
    truth_length [B] label counts incl. <S/E>).  -> i64 0-d tensors (errors of the 1-best, sum over utterances of the
    fewest errors in the n-best, reference tokens): eval.py's false_tokens, top_n_false_tokens and total_tokens.  Both
    sides of the comparison are at most 1023 tokens long.  Word merging (-p2w) is not applied."""
    B, K, W = ids.shape
    dev = ids.device
    ext = torch.cat((ids.long(), torch.full((B, K, 1), EOS, dtype=torch.int64, device=dev)), dim=2)
    if lengths is not None:
        ext = torch.where(torch.arange(W + 1, device=dev) >= lengths[..., None], EOS, ext)
    n = (ext == EOS).int().argmax(dim=2).to(torch.int32)                         # the first <S/E>, as second_pass_rows cuts
    ref_len = (truth_length.to(dev).to(torch.int32) - 1).contiguous()
    err = ops.edit_distance(ids.reshape(B * K, W), n.view(-1), truth[:, 1:].to(dev), ref_len, K).view(B, K).long()
    return err[:, 0].sum(), err.min(dim=1).values.sum(), ref_len.long().sum()


def rescore_nbest(ids, scores, scorers, weight, nbest, width=None, pad=EOS, lengths=None, rows=None):
    """N-best rescoring (DESIGN.md 4.10): first-pass ids [B, K, W] (cut as second_pass_rows does) with scores f32 [B, K];
    scorers: functions (inputs i64 [B*K, Lp], targets i32 [B*K, Lp], K, Lp) -> token log-probs f32 [B*K, Lp] of one
    second-pass model each.  s = first-pass score + weight * sum of the models' sums; ranked per utterance by descending s,
    ties in first-pass order, duplicates last with -inf.  -> ops.nbest_rescore's (ids i64 [B, nbest, width or Lp] padded
    with `pad`, lengths i32 [B, nbest], scores f32 [B, nbest]).  rows: second_pass_rows(ids, lengths) when the caller has
    it already."""
    B, K, _ = ids.shape
    inputs, targets, n, Lp = rows if rows is not None else second_pass_rows(ids, lengths)
    flat = targets.view(B * K, Lp)
    tok_lp = torch.stack([f(inputs, flat, K, Lp).reshape(B, K, Lp) for f in scorers])
    return ops.nbest_rescore(targets, n, scores.float().contiguous(), tok_lp.contiguous(), weight, nbest, width or Lp, pad)


def ctc_rescoring_terms(head, mem, mem_len, B, T2, V, targets, scores):
    """The joint-CTC head's part of apply_ctc_rescoring (DESIGN.md 4.18): log p_ctc(y <S/E> | x) of each first-pass
    hypothesis (targets i32 [B, K, Lp] as second_pass_rows builds them) over the head's log-probs of memory bf16 [B*T2, D].
    -> (first-pass scores f32 [B, K] with -inf where the CTC score is -inf, the CTC term as rescore_nbest's token log-probs
    f32 [B*K, Lp]: the sequence score at position 0, zeros elsewhere and for the -inf rows).  Moving the -inf of a
    hypothesis without a CTC alignment into its first-pass score makes its rescored score -inf whatever the weight (w * -inf
    would be NaN at w = 0 and +inf below), so it ranks after every hypothesis with one, in first-pass order."""
    B, K, Lp = targets.shape
    ctc = ops.ctc_nbest_score(ops.log_softmax(head.logits_bf16(mem), V), B, T2, mem_len, targets, head.blank)
    feasible = ctc > float('-inf')
    tok = torch.zeros(B * K, Lp, dtype=torch.float32, device=ctc.device)
    tok[:, 0] = torch.where(feasible, ctc, 0.0).view(-1)
    return torch.where(feasible, scores, float('-inf')), tok


def check_lm_rescoring(who, lm, vocab_size):
    if lm is None:
        raise ValueError(f'{who}: apply_lm_rescoring needs an lm')
    if getattr(lm, 'model_type', None) not in ('transformer_lm', 'recurrent_lm'):
        raise NotImplementedError(f'{who}: LM rescoring is implemented for the Transformer and the recurrent LM '
                                  '(opentransformer_b200.lm)')
    if lm.vocab_size != vocab_size:
        raise ValueError(f'{who}: the LM has {lm.vocab_size} tokens and the model {vocab_size}: rescoring needs one vocabulary')


def check_lm_fusion(who, lm, vocab_size):
    if getattr(lm, 'model_type', None) not in ('transformer_lm', 'recurrent_lm'):
        raise NotImplementedError('shallow fusion is implemented for the Transformer and the recurrent LM '
                                  '(opentransformer_b200.lm)')
    if lm.vocab_size != vocab_size:
        raise ValueError(f'{who}: the LM has {lm.vocab_size} tokens and the model {vocab_size}: shallow fusion needs one '
                         'vocabulary')


def check_max_len(who, max_len):
    """The KV-cached search takes max_len <= 1023 (otb_decode_self_attn); past 128 it runs on the per-step graph path."""
    if max_len > ops.DECODE_MAX_LEN:
        raise ValueError(f'{who}: max_len must be at most {ops.DECODE_MAX_LEN}, got {max_len}')


def ctc_decode(logits, lengths, B, T2, V, blank, mode, beam_width):
    """CTC decoding of a CTC head's logits f32 [B*T', ld] (CTCRecognizer; SpeechToTextRecognizer's first pass under
    apply_rescoring): otb_ctc_frame_topk, then the greedy collapse (otb_ctc_greedy, mode 'greedy') or the prefix beam search
    over each frame's 40 best tokens (otb_ctc_prefix_beam, mode 'beam').  -> (ids i64 [B, nbest, T'] best first, 0 after
    each hypothesis' end; lengths i32 [B, nbest]; scores f32 [B, nbest]); nbest is 1 in greedy mode and beam_width in beam
    mode."""
    if mode == 'greedy':
        lp, tok = ops.ctc_frame_topk(logits, B, T2, V, lengths, 1)
        ids, n, sc = ops.ctc_greedy(lp, tok, B, T2, lengths, blank)
        return ids.long().view(B, 1, T2), n.view(B, 1), sc.view(B, 1)
    lp, tok = ops.ctc_frame_topk(logits, B, T2, V, lengths, min(CTC_CUTOFF_TOP_N, V))
    ids, n, sc = ops.ctc_prefix_beam(lp, tok, B, T2, lengths, beam_width, blank)
    return ids.long(), n, sc


class BeamDecoder:
    """KV-cached incremental decoder + device-side beam search for one (batch, beam, T, max_len) shape.

    Buffers are allocated once; one decode step (decoder on the newest token -> log-softmax -> beam
    kernel) is self.step, a graphs.CapturedStep: the first step runs eagerly, is captured, and every later step replays it
    (a new weight pack, the decoder's or the fused LM's, captures again).

    ctc = (assistor, weight, P) adds the CTC prefix term of joint CTC/attention decoding (DESIGN.md 4.9): setup() takes
    the head's log-probs, and a step scores each hypothesis' P best tokens with
    (1 - weight) logp_att + weight (psi(g c) - psi(g)) + lm_weight lm before the beam kernel selects among the `beam`
    best of them.  The persistent kernel does not take the term, so it is off then.

    lm = (lm, weight) fuses a language model (speech2text.py:101-105): every step computes its log-probs into lm_logp
    [N, V] inside the same step (and the same captured graph) before the fused log-softmax/top-k adds weight * lm_logp.
    The Transformer LM runs its newest position against a KV cache [blocks, max_len, N, d_lm] addressed by the search's own
    ancestry and step counter, so beam pruning reorders it for free; the recurrent LM reads the newest token from a zero
    state, as the reference does (cache['lm'] = None at every step).  The persistent kernel does not take an LM, so it is
    off then.

    sample=True turns the search into ancestral sampling (DESIGN.md 4.11): the `beam` rows of an utterance all start live
    at BOS with score 0, and each step draws every live row's next token from the decoder's softmax (ops.sample_step, the
    Gumbel-max trick on a counter hash of (seed, step, row, token)) in place of the log-softmax / top-k / beam kernels.  Rows
    are never reordered, and a row's score is the log-probability of its sample.  The seed is the i32 device scalar
    `self.seed`, read by every replay of the captured step.  Not with an LM or a CTC term, and never on the persistent
    kernel.
    """

    def __init__(self, decoder, batch, beam, T, max_len, device, use_graph=True, persistent=False, keep_logp=None, ctc=None,
                 lm=None, sample=False):
        check_max_len('BeamDecoder', max_len)
        if sample and (lm is not None or ctc is not None):
            raise NotImplementedError('BeamDecoder: sampling draws from the attention decoder alone; sampling with a fused LM '
                                      'or a CTC term is not implemented')
        if lm is not None:
            check_lm_fusion('BeamDecoder', lm[0], decoder.vocab_size)
        self.dec = decoder
        self.B, self.beam, self.T, self.Lmax = batch, beam, T, max_len
        self.N = batch * beam
        self.device = device
        d, nl = decoder.d_model, len(decoder.blocks)
        self.state = ops.BeamState(batch, beam, max_len, device)
        self.kc = torch.zeros(nl, max_len, self.N, d, dtype=ops.BF16, device=device)
        self.vc = torch.zeros(nl, max_len, self.N, d, dtype=ops.BF16, device=device)
        self.kvx = torch.zeros(nl, batch * T, 2 * d, dtype=ops.BF16, device=device)  # cross K|V per utterance
        self.mem_len = torch.zeros(batch, dtype=torch.int32, device=device)
        self.table = ops.sinusoid_table(max_len + 1, d, 0, device)
        self.logits = torch.zeros(self.N, decoder.ld_logits, dtype=torch.float32, device=device)
        self.logp = torch.zeros(self.N, decoder.vocab_size, dtype=torch.float32, device=device)
        self.topk_val = torch.zeros(self.N, beam, dtype=torch.float32, device=device)
        self.topk_idx = torch.zeros(self.N, beam, dtype=torch.int32, device=device)
        # eager (test / debug) mode also materialises the full log-probs; keep_logp=True does so on the graph path (parity traces)
        self.keep_logp = (not use_graph) if keep_logp is None else bool(keep_logp)
        self.use_graph = use_graph
        self.step = CapturedStep(self._step_kernels, self._packs, use_graph)     # one decode step
        self.lm_logp = None
        self.lm_weight = 0.0
        self.lm = self.lm_cache = self._lstm_bar = None
        if lm is not None:
            self.lm, weight = lm
            self.lm_weight = float(weight)
            self.lm_logp = torch.zeros(self.N, decoder.vocab_size, dtype=torch.float32, device=device)
            if self.lm.model_type == 'transformer_lm':
                self.lm_cache = LMCache(self.lm, self.N, max_len, anc=self.state.anc, step_ptr=self.state.step_ptr)
            else:
                self.lm._check_device(device)
                # the recurrence kernel's grid barrier, allocated here and not inside the capture (one step never syncs on it)
                self._lstm_bar = torch.zeros(2, dtype=torch.int32, device=device)
        if decoder.pos_emb.scale_learnable:
            raise NotImplementedError('decoder with learnable positional scale')
        self.ctc = self.ctc_head = None
        self.ctc_weight = 0.0
        if ctc is not None:
            self.ctc_head, weight, P = ctc
            self.ctc_weight = float(weight)
            self.ctc = ops.CTCPrefixState(batch, beam, T, decoder.vocab_size, P, device, blank=self.ctc_head.blank)
        # persistent path: the whole loop in ONE launch (csrc/decode_group.cu: row groups of <= 128 hypotheses x 16 CTAs,
        # wgmma GEMMs, group-local barriers) when the configuration is the shipped one (post-norm GLU decoder, d_model 256,
        # 4 heads, d_ff 2048, <= 256 memory frames); anything else takes the per-step graph.
        self.sample = bool(sample)
        self.seed = torch.zeros(1, dtype=torch.int32, device=device) if self.sample else None
        self.persistent = (bool(persistent) and self.ctc is None and self.lm is None and not self.sample
                           and self.mega_supported())
        self._mega_model = None
        self._mega_sig = None
        self._ws = None

    def mega_supported(self):
        dec = self.dec
        groups = -(-self.B // max(1, 128 // self.beam))
        ok = (dec.d_model == 256 and dec.n_heads == 4 and not dec.normalize_before and 1 <= len(dec.blocks) <= 8
              and self.beam <= 16 and self.Lmax <= 128 and dec.vocab_size >= 16 and self.T <= 256
              and groups * 16 <= ops.num_sms())
        for blk in dec.blocks:
            ff = blk.feed_forward
            ok = ok and ff.activation == 'glu' and ff.w_2.in_features == 2048 and not blk.normalize_before
            ok = ok and all(m.bias is not None for m in (blk.slf_attn.qvk_proj, blk.slf_attn.output_proj, blk.src_attn.q_proj,
                                                         blk.src_attn.output_proj, ff.w_1, ff.w_2))
        return bool(ok)

    def _mega(self):
        """otb_mega_model over the packed bf16 weights (rebuilt when the pack changes)."""
        pk = self.dec.packed()
        if self._mega_model is None or self._mega_sig is not pk:
            from ._lib import MegaModelC
            m = MegaModelC()
            m.n_layers, m.d_model, m.n_heads = len(self.dec.blocks), self.dec.d_model, self.dec.n_heads
            m.d_ff, m.vocab = self.dec.blocks[0].feed_forward.w_2.in_features, self.dec.vocab_size
            m.emb, m.wout = pk['emb'].data_ptr(), pk['wout'].data_ptr()
            m.bout = pk['bout'].data_ptr() if pk['bout'] is not None else None
            m.pe = self.table.data_ptr()
            m.ln_eps = 1e-5
            for l, p in enumerate(pk['blocks']):
                ly = m.layers[l]
                f = p['ffn']
                for name, t in (('wqkv', p['wqkv']), ('wo', p['wo']), ('wq', p['wq']), ('wo2', p['wo2']), ('w1', f['w1']),
                                ('w2', f['w2']), ('bqkv', p['bqkv']), ('bo', p['bo']), ('bq', p['bq']), ('bo2', p['bo2']),
                                ('b1', f['b1']), ('b2', f['b2']), ('g1', p['ln1'][0]), ('be1', p['ln1'][1]),
                                ('g2', p['ln2'][0]), ('be2', p['ln2'][1]), ('g3', p['ln3'][0]), ('be3', p['ln3'][1])):
                    setattr(ly, name, t.data_ptr())
            self._mega_model, self._mega_sig = m, pk
        return self._mega_model

    def run_persistent(self, max_steps, dbg_logp=None, dbg_scores=None):
        """All steps in ONE launch; no host round trip (ctrl[0] = executed steps is read by the caller)."""
        if self._ws is None:
            self._ws = ops.decode_persistent_workspace(self.N, len(self.dec.blocks), self.Lmax, self.B, self.beam,
                                                       self.dec.vocab_size, self.device)
        ops.decode_persistent(self._mega(), self.kvx, self.mem_len, self.kc, self.vc, self.state, self.B, self.T, max_steps,
                              self._ws, dbg_logp, dbg_scores)

    def setup(self, memory_bf16, mem_len):
        """Project cross-attention K/V once per utterance and reset the search state (with a CTC term: the head's
        log-probs of every frame and the prefix state of the empty hypothesis)."""
        pk = self.dec.packed()
        self.mem_len.copy_(mem_len)
        for l, p in enumerate(pk['blocks']):
            ops.linear(memory_bf16, p['wkv'], p['bkv'], out=self.kvx[l])
        self.state.init()
        if self.sample:
            self.state.scores.zero_()           # every row starts live (the beam's init leaves rows 1.. at -inf)
        if self.ctc is not None:
            ops.log_softmax(self.ctc_head.logits_bf16(memory_bf16), self.dec.vocab_size, out=self.ctc.lp)
            self.ctc.init(self.mem_len)

    def _packs(self):
        return (self.dec.packed(),) if self.lm is None else (self.dec.packed(), self.lm._pack.get())

    def _lm_step(self):
        """The fused LM's log-probs of every hypothesis' next token -> lm_logp."""
        lm, st = self.lm, self.state
        pk = lm._pack.get()
        if self.lm_cache is not None:
            lm.cached_log_probs(pk, st.last_tok, self.lm_cache, out=self.lm_logp)
            return
        # lm_log_probs' kernels for the RNN LM (predict of the newest token, zero state)
        x, _, _, _ = lm._run(st.last_tok.view(1, self.N), pk, barrier=self._lstm_bar)
        ops.log_softmax(lm._logits(x, pk), lm.vocab_size, out=self.lm_logp)

    def _step_kernels(self):
        dec, st = self.dec, self.state
        pk = dec.packed()
        if self.lm is not None:
            self._lm_step()
        x = ops.embed_posenc(st.last_tok, pk['emb'], self.table, self.N, dec.d_model, step_ptr=st.step_ptr)
        x = dec.decode_cached_bf16(pk, x, self.kc, self.vc, st.anc, st.step_ptr, self.kvx, self.mem_len, self.beam, self.T)
        ops.linear(x, pk['wout'], pk['bout'], out=self.logits)
        if self.sample:
            ops.sample_step(self.logits, dec.vocab_size, st, self.seed)
            return
        out_logp = self.logp if self.keep_logp else None
        if self.ctc is None:
            ops.logsoftmax_topk(self.logits, dec.vocab_size, self.beam, self.lm_logp, self.lm_weight,
                                out_val=self.topk_val, out_idx=self.topk_idx, out_logp=out_logp)
            st.step_topk(self.topk_val, self.topk_idx)
            return
        ctc = self.ctc
        ops.logsoftmax_topk(self.logits, dec.vocab_size, ctc.P, self.lm_logp, self.lm_weight,
                            out_val=ctc.cand_val, out_idx=ctc.cand_id, out_logp=out_logp)
        ctc.score(st, self.mem_len, self.ctc_weight, self.topk_val, self.topk_idx, self.lm_logp, self.lm_weight)
        st.step_topk(self.topk_val, self.topk_idx)
        ctc.advance(st, self.mem_len)

    @property
    def graph(self):
        """The captured decode step (None until the first step of the graph path)."""
        return self.step.graph

    def _read_ctrl(self):
        """{step, done, ...} of the search state on the host (graphs.read_device)."""
        return read_device(self.state.ctrl)

    def run(self, max_steps, poll_every=8):
        """Run up to max_steps decode steps; stops early once the device reports every hypothesis ended
        (speech2text.py:66-67).  Steps launched after the end are no-ops on the search state.
        (A sync-free variant -- the flag copied asynchronously to pinned memory and inspected one poll later -- lets
        free-running lanes fall into lockstep and queue for the same SMs, whereas this 4-byte poll staggers them.)"""
        if self.persistent and self.lm_logp is None:
            self.run_persistent(max_steps)
            return int(self._read_ctrl()[0])
        for i in range(max_steps):
            self.step()
            if (i + 1) % poll_every == 0 and i + 1 < max_steps:
                if int(self._read_ctrl()[1]):
                    break
        return int(self._read_ctrl()[0])


class SpeechToTextRecognizer(Recognizer):
    """otrans/recognize/speech2text.py:6-93 on the CUDA path."""

    def __init__(self, model, lm=None, lm_weight=0.1, ctc_weight=0.0, beam_width=5, nbest=1, max_len=50,
                 idx2unit=None, penalty=0, lamda=5, ngpu=1, apply_cache=False, use_graph=True, persistent=None,
                 ctc_candidates=None, apply_rescoring=False, apply_lm_rescoring=False, rescore_weight=1.0, max_decoders=None,
                 apply_ctc_rescoring=False):
        """ctc_weight w > 0: joint CTC/attention decoding (DESIGN.md 4.9).  Each hypothesis' ctc_candidates best tokens by
        the attention (+ LM) score (default min(16, 2 beam_width), between beam_width and 16) are scored
        (1 - w) logp_att + w (psi(g c) - psi(g)) + lm_weight lm with the CTC prefix score psi of the model's joint-CTC head,
        and the search goes on with the beam_width best of them.  The model must have the head (params['ctc_weight'] > 0).

        N-best rescoring (DESIGN.md 4.10; eval.py's -resc / -lm_resc / -rw): each hypothesis' score becomes
        s = first-pass score + rescore_weight * (sum of its second-pass log-probs), and the nbest best by s are returned.
        apply_rescoring: the first pass is the CTC prefix beam search (beam_width hypotheses) over the joint-CTC head, the
        second pass the attention decoder; no attention beam search runs.  apply_lm_rescoring: the LM is not fused into the
        search (the persistent decode kernel stays eligible) but scores all beam_width hypotheses of the first pass.
        apply_ctc_rescoring (DESIGN.md 4.18): the attention beam search runs as without it (on the persistent kernel when
        eligible) and the joint-CTC head's log p_ctc(y <S/E> | x) of each of its beam_width hypotheses is a second-pass
        score; with apply_lm_rescoring both scores add before rescore_weight.  A hypothesis the head cannot emit (no CTC
        alignment) scores -inf and ranks after the others, in first-pass order.

        max_decoders: at most this many BeamDecoders (one per batch geometry: batch, encoder frames; each owns its KV caches
        and search buffers) are kept, least recently used first out; None keeps one per geometry seen."""
        check_max_len('SpeechToTextRecognizer', max_len)
        has_head = getattr(model, 'ctc_weight', 0.0) > 0.0
        if apply_rescoring and not has_head:
            raise ValueError('SpeechToTextRecognizer: apply_rescoring needs the joint-CTC head: this model has ctc_weight 0')
        if apply_rescoring and ctc_weight > 0.0:
            raise ValueError('SpeechToTextRecognizer: apply_rescoring (CTC first pass, attention second) and ctc_weight > 0 '
                             '(the CTC term inside the attention search) are two uses of the joint-CTC head; choose one')
        if apply_ctc_rescoring and not has_head:
            raise ValueError('SpeechToTextRecognizer: apply_ctc_rescoring needs the joint-CTC head: this model has ctc_weight 0')
        if apply_ctc_rescoring and ctc_weight > 0.0:
            raise ValueError('SpeechToTextRecognizer: apply_ctc_rescoring (the CTC head re-ranking the attention n-best) and '
                             'ctc_weight > 0 (the CTC term inside the attention search) are two uses of the joint-CTC head; '
                             'choose one')
        if apply_ctc_rescoring and apply_rescoring:
            raise ValueError('SpeechToTextRecognizer: apply_ctc_rescoring re-ranks the attention search\'s n-best, and under '
                             'apply_rescoring the first pass is the CTC head\'s own beam search; choose one')
        if apply_rescoring and not 1 <= beam_width <= 16:
            raise NotImplementedError(f'SpeechToTextRecognizer: the CTC prefix beam search of apply_rescoring takes beam_width '
                                      f'1..16, got {beam_width}')
        if apply_lm_rescoring:
            check_lm_rescoring('SpeechToTextRecognizer', lm, model.decoder.vocab_size)
        elif lm is not None:
            check_lm_fusion('SpeechToTextRecognizer', lm, model.decoder.vocab_size)
        if not 0.0 <= ctc_weight <= 1.0:
            raise ValueError(f'SpeechToTextRecognizer: ctc_weight must be in [0, 1], got {ctc_weight}')
        if ctc_weight > 0.0 and getattr(model, 'ctc_weight', 0.0) <= 0.0:
            raise ValueError('SpeechToTextRecognizer: ctc_weight > 0 needs the joint-CTC head: this model has ctc_weight 0')
        if ctc_candidates is None:
            ctc_candidates = max(beam_width, min(ops.CTC_PREFIX_MAX_CANDIDATES, 2 * beam_width))
        if ctc_weight > 0.0 and not beam_width <= ctc_candidates <= ops.CTC_PREFIX_MAX_CANDIDATES:
            raise ValueError(f'SpeechToTextRecognizer: ctc_candidates must be in [beam_width = {beam_width}, '
                             f'{ops.CTC_PREFIX_MAX_CANDIDATES}], got {ctc_candidates}')
        super().__init__(model, idx2unit, lm, lm_weight, ngpu)
        self.beam_width, self.max_len, self.nbest = beam_width, max_len, nbest
        self.penalty, self.lamda = penalty, lamda
        self.ctc_weight, self.lm_weight, self.ctc_candidates = ctc_weight, lm_weight, ctc_candidates
        self.attn_weights = {}
        self.apply_cache = False
        self.use_graph = use_graph
        # None = automatic: the persistent decode kernel (one launch per batch, csrc/decode_group.cu) whenever the decoder,
        # the batch geometry and the options (no CTC term, no LM fusion) fit it; False forces the per-step CUDA-graph path
        self.persistent = True if persistent is None else bool(persistent)
        self.apply_rescoring, self.apply_lm_rescoring = bool(apply_rescoring), bool(apply_lm_rescoring)
        self.apply_ctc_rescoring = bool(apply_ctc_rescoring)
        self.rescore_weight = float(rescore_weight)
        self._decoders = {}
        if max_decoders is not None and max_decoders < 1:
            raise ValueError(f'SpeechToTextRecognizer: max_decoders must be >= 1 or None, got {max_decoders}')
        self.max_decoders = max_decoders

    # ---- reference-facing seams -------------------------------------------------------------
    def encode(self, inputs, inputs_mask, cache=None):
        """-> (memory, memory_mask, cache, attention weights): the encoder's attn_weights dict when
        model.encoder.return_attn_weights is set, else {}."""
        mem, mem_len, B, T2 = self._encode_bf16(inputs, inputs_mask)
        memory = mem.float().view(B, T2, -1)
        maps = self.attn_weights['encoder'] if self.model.encoder.return_attn_weights else {}
        return memory, self.model.frontend.output_mask(inputs_mask), {'frontend': None}, maps

    def decode(self, preds, memory, memory_mask, cache=None):
        return self.model.decoder.inference(preds, memory, memory_mask, cache)

    def decode_step(self, preds, memory, memory_mask, cache, scores, flag):
        """One reference-style step on caller-owned tensors (speech2text.py:95-153): decoder.inference + the CUDA beam
        kernel.  With cache['decoder'] = model.decoder.init_cache(memory, mask, max_len, beam) the decoder runs KV-cached
        (one token per call) and the cache is reordered by the surviving hypotheses' parents -- the feature the reference
        left as a stub (decoder/transformer.py:188-203, reselect_hidden* :195-218); with None it recomputes the full prefix
        like the reference.  The fast path used by recognize() is BeamDecoder; the CTC term of joint decoding exists there
        only, so a recognizer with ctc_weight > 0 refuses this seam."""
        from .modules import DecoderCache
        if self.ctc_weight > 0.0:
            raise NotImplementedError('decode_step is attention-only: joint CTC/attention decoding (ctc_weight > 0) runs in '
                                      'recognize() / recognize_ids()')
        n = scores.size(0)
        batch = n // self.beam_width
        dcache = cache.get('decoder') if isinstance(cache, dict) else None
        lcache = cache.get('lm') if isinstance(cache, dict) else None
        log_probs, dcache, _ = self.decode(preds, memory, memory_mask, dcache)
        st = ops.BeamState(batch, self.beam_width, 1, scores.device)
        st.init()
        st.scores.copy_(scores.view(-1))
        st.flag.copy_(flag.view(-1).to(torch.uint8))
        lm_logp, lm_w = None, 0.0
        if self.lm is not None and self.lm_weight:
            if isinstance(lcache, LMCache):
                lm_logp = self.lm.predict(preds, True, lcache).squeeze(1)
            else:
                lm_logp = lm_log_probs(self.lm, preds)
            lm_w = float(self.lm_weight)
        st.step(log_probs.contiguous(), log_probs.shape[-1], lm_logp, lm_w)
        parent = st.par_hist[0].long()
        tok = st.tok_hist[0].long()
        if isinstance(dcache, DecoderCache):
            dcache.reorder(parent)
        if lm_logp is not None and isinstance(lcache, LMCache):
            lcache.reorder(parent)
        preds_symbol = torch.cat((preds.index_select(0, parent), tok.view(-1, 1)), dim=1)
        return preds_symbol, cache, st.scores.view(-1, 1).clone(), (tok == EOS).view(-1, 1)

    # ---- fast path ------------------------------------------------------------------------------
    def _encode_bf16(self, inputs, inputs_mask):
        """The encoder pass of every path.  With model.encoder.return_attn_weights set it also fills self.attn_weights
        as the reference's recognize does (recognize/speech2text.py:43-47): {'encoder': the encoder's attn_weights dict,
        'decoder': []}; otherwise attn_weights stays {}."""
        enc = self.model.encoder
        if not enc.return_attn_weights:
            return self.model.encode_bf16(inputs, inputs_mask)
        sink = []
        out = self.model.encode_bf16(inputs, inputs_mask, attn_sink=sink)
        self.attn_weights = {'encoder': encoder_attn_weights(len(enc.blocks), sink), 'decoder': []}
        return out

    def _decoder_for(self, B, T2, device, samples=0):
        # the CTC weight and candidate count, the fused LM's weights and lm_weight are launch arguments that a captured step
        # bakes in; samples > 0: a sampling decoder of that many rows per utterance, kept apart from the beam decoders
        ctc = (self.model.assistor, self.ctc_weight, self.ctc_candidates) if self.ctc_weight > 0.0 else None
        lm = (self.lm, float(self.lm_weight)) if self._lm_fused() else None
        rows = samples or self.beam_width
        key = (B, rows, T2, self.max_len, device.index, ctc[1:] if ctc else None, lm, 'sample' if samples else 'beam')
        return lru_get(self._decoders, key, self.max_decoders, lambda: BeamDecoder(
            self.model.decoder, B, rows, T2, self.max_len, device, self.use_graph, persistent=self.persistent, ctc=ctc, lm=lm,
            sample=bool(samples)))

    def _lm_fused(self):
        """The LM enters the search by shallow fusion (it rescores the n-best instead under apply_lm_rescoring)."""
        return self.lm is not None and not self.apply_lm_rescoring

    def _search(self, inputs, inputs_mask):
        """Encoder pass, search and (when asked) rescoring -> (recognize_ids' return, memory bf16 [B*T', D], lengths i32 [B],
        the BeamDecoder or None when the first pass is the CTC prefix beam search)."""
        mem, mem_len, B, T2 = self._encode_bf16(inputs, inputs_mask)
        scorers = []
        if self.apply_rescoring:
            dec = self.model.decoder
            scorers.append(lambda x, y, K, Lp: ops.token_logprob(dec.score_bf16(x, mem, mem_len, B, K, Lp, T2), dec.vocab_size,
                                                                 y.reshape(-1)))
        if self.apply_lm_rescoring:
            scorers.append(lambda x, y, K, Lp: lm_token_logprob(self.lm, x, y))
        nbest = min(self.nbest, self.beam_width)
        if self.apply_rescoring:
            ids, n, sc = ctc_decode(self.model.assistor.logits_bf16(mem), mem_len, B, T2, self.model.decoder.vocab_size,
                                    self.model.assistor.blank, 'beam', self.beam_width)
            preds, _, scores = rescore_nbest(ids, sc, scorers, self.rescore_weight, nbest, lengths=n)
            return (preds, scores, preds.shape[2]), mem, mem_len, None
        bd = self._decoder_for(B, T2, inputs.device)
        bd.setup(mem, mem_len)
        steps = bd.run(self.max_len)
        if not scorers and not self.apply_ctc_rescoring:
            preds, scores = bd.state.finalize(self.penalty, self.lamda, self.nbest)
            return (preds[:, :, :steps], scores, steps), mem, mem_len, bd
        preds, scores = bd.state.finalize(self.penalty, self.lamda, self.beam_width)
        preds, rows = preds[:, :, :steps], None
        if self.apply_ctc_rescoring:
            rows = second_pass_rows(preds)
            scores, ctc_tok = ctc_rescoring_terms(self.model.assistor, mem, mem_len, B, T2, self.model.decoder.vocab_size,
                                                  rows[1], scores)
            scorers.append(lambda x, y, K, Lp: ctc_tok)
        preds, _, scores = rescore_nbest(preds, scores, scorers, self.rescore_weight, nbest, width=steps, rows=rows)
        return (preds, scores, steps), mem, mem_len, bd

    def recognize_ids(self, inputs, inputs_mask):
        """-> (nbest ids i64 [B,nbest,steps], scores f32 [B,nbest], steps)"""
        with torch.no_grad():
            return self._search(inputs, inputs_mask)[0]

    def recognize_spans(self, inputs, inputs_mask):
        """recognize_ids, plus where each token of the 1-best lies: the 1-best up to and including its closing <S/E> (one is
        appended to a hypothesis that reached max_len without it; the head is trained on the closing <S/E> as a label) is
        force-aligned (otb_ctc_align) against the joint-CTC head's log-probs of the same encoder pass.  Any ctc_weight, 0
        included, but the model must have the head.  -> (ids, scores, steps as recognize_ids; spans i32 [B, steps + 1, 2]
        [start, end) in encoder frames of the 1-best's tokens, -1 past its closing <S/E> and throughout where the
        utterance has too few frames for it), on the device.  model.encoder_frames_to_input converts the spans."""
        if getattr(self.model, 'ctc_weight', 0.0) <= 0.0:
            raise ValueError('SpeechToTextRecognizer.recognize_spans needs the joint-CTC head: this model has ctc_weight 0')
        with torch.no_grad():
            (ids, scores, steps), mem, mem_len, bd = self._search(inputs, inputs_mask)
            B, V = ids.shape[0], self.model.decoder.vocab_size
            lp = bd.ctc.lp if bd is not None and bd.ctc is not None else ops.log_softmax(self.model.assistor.logits_bf16(mem), V)
            best = torch.cat((ids[:, 0], torch.full((B, 1), EOS, dtype=ids.dtype, device=ids.device)), dim=1)
            n_tok = ((best == EOS).int().argmax(dim=1) + 1).to(torch.int32)
            _, _, spans, _ = ops.ctc_align(lp.view(B, -1, V), mem_len, best, n_tok, blank=self.model.assistor.blank)
        return ids, scores, steps, spans

    def recognize(self, inputs, inputs_mask):
        preds, scores, _ = self.recognize_ids(inputs, inputs_mask)
        return self.nbest_translate(preds), scores

    def sample_ids(self, inputs, inputs_mask, num_samples, seed=0):
        """Draw num_samples (1..16) hypotheses per utterance from the attention decoder, y ~ P(y | x), by ancestral sampling
        at temperature 1 (DESIGN.md 4.11): up to max_len tokens each, one captured step per token, the samples drawn
        independently and with replacement.  seed: an int, or an i32 device tensor of one element (read on the device, so
        a caller can advance it without a host synchronisation); the same seed and weights give the same samples.
        -> (ids i64 [B, num_samples, steps] in sample order, <S/E> after each sample's end, as recognize_ids pads; lengths
        i32 [B, num_samples], the tokens before <S/E>; log-probs f32 [B, num_samples], the sum of each sample's token
        log-probs, its closing <S/E> included), on the device.  Not with LM fusion, a CTC term (ctc_weight > 0) or
        apply_rescoring (NotImplementedError)."""
        if self._lm_fused():
            raise NotImplementedError('sample_ids: sampling from the LM-fused distribution is not implemented; build the '
                                      'recognizer without lm (or with apply_lm_rescoring)')
        if self.ctc_weight > 0.0:
            raise NotImplementedError('sample_ids: sampling from the joint CTC/attention distribution (ctc_weight > 0) is not '
                                      'implemented')
        if self.apply_rescoring:
            raise NotImplementedError('sample_ids: under apply_rescoring the first pass is the CTC prefix beam search; '
                                      'sampling draws from the attention decoder alone')
        if not isinstance(num_samples, int) or not 1 <= num_samples <= 16:
            raise ValueError(f'sample_ids: num_samples must be in 1..16, got {num_samples}')
        K = num_samples
        with torch.no_grad():
            mem, mem_len, B, T2 = self._encode_bf16(inputs, inputs_mask)
            bd = self._decoder_for(B, T2, inputs.device, samples=K)
            bd.setup(mem, mem_len)
            if torch.is_tensor(seed):
                bd.seed.copy_(seed.reshape(1))
            else:
                bd.seed.fill_((int(seed) + 2 ** 31) % 2 ** 32 - 2 ** 31)         # the seed's 32 bits as an i32
            steps = bd.run(self.max_len)
            ids = bd.state.reconstruct(steps)[:, 1:].reshape(B, K, steps)
            lengths = (ids != EOS).sum(dim=2, dtype=torch.int32)      # an ended row emits only <S/E>
            return ids, lengths, bd.state.scores.view(B, K).clone()


CTC_CUTOFF_TOP_N = 40      # ctcdecode's cutoff_top_n default (cutoff_prob 1.0), which recognize/ctc.py:20-24 leaves in place


class CTCRecognizer(Recognizer):
    """otrans/recognize/ctc.py:7-76 on the CUDA path: CTCModel.inference's head logits -> otb_ctc_frame_topk -> the greedy
    collapse (otb_ctc_greedy, mode 'greedy') or the CTC prefix beam search (otb_ctc_prefix_beam, mode 'beam': ctcdecode's
    search without a scorer, over each frame's 40 best tokens).  `lm` is used only by apply_lm_rescoring and lm_fusion, as
    the reference never uses it; `alpha` is ignored, and `beta` too unless lm_fusion is on, as ctcdecode ignores them
    without a scorer; an n-gram LM (`ngram_lm`, KenLM) is refused.

    apply_lm_rescoring (beam mode): the prefix beam search's n-best is re-ranked by
    s = prefix log-probability + rescore_weight * log P_lm(y <S/E>) (DESIGN.md 4.10).

    lm_fusion (beam mode, off by default): the LM is ctcdecode's scorer inside the search (DESIGN.md 4.19).  Extending a
    prefix by token c adds lm_weight * log p_lm(c | <S/E>, prefix) + beta; the scores are those fused totals.  The search
    runs one frame per replay of a captured CUDA graph (use_graph=False: the same kernels launched one by one)."""

    def __init__(self, model, lm=None, lm_weight=0.1, ngram_lm=None, beam_width=5, idx2unit=None, ngpu=1, mode='greedy',
                 alpha=0.1, beta=0.0, apply_lm_rescoring=False, rescore_weight=1.0, lm_fusion=False, use_graph=True):
        if lm_fusion:
            if lm is None:
                raise ValueError('CTCRecognizer: lm_fusion needs an lm')
            if mode != 'beam':
                raise ValueError("CTCRecognizer: lm_fusion fuses the LM into the prefix beam search; use mode='beam'")
            if apply_lm_rescoring:
                raise ValueError('CTCRecognizer: lm_fusion and apply_lm_rescoring would count the same LM twice; choose one')
            check_lm_fusion('CTCRecognizer', lm, model.vocab_size)
        if ngram_lm is not None:
            raise NotImplementedError('CTCRecognizer: n-gram LM scoring (KenLM) is not implemented; use ngram_lm=None')
        if mode not in ('greedy', 'beam'):
            raise ValueError(f"CTCRecognizer: mode must be 'greedy' or 'beam', got {mode!r}")
        if mode == 'beam' and not 1 <= beam_width <= 16:
            raise NotImplementedError(f'CTCRecognizer: the prefix beam search takes beam_width 1..16, got {beam_width}')
        if apply_lm_rescoring:
            if mode == 'greedy':
                raise ValueError("CTCRecognizer: apply_lm_rescoring re-ranks an n-best; the greedy mode has one hypothesis, "
                                 "use mode='beam'")
            check_lm_rescoring('CTCRecognizer', lm, model.vocab_size)
        super().__init__(model, idx2unit, lm, lm_weight, ngpu)
        self.beam_width, self.mode = beam_width, mode
        self.alpha, self.beta = alpha, beta
        self.apply_lm_rescoring, self.rescore_weight = bool(apply_lm_rescoring), float(rescore_weight)
        self.lm_fusion, self.use_graph = bool(lm_fusion), bool(use_graph)
        self._searches = {}

    def _check_frames(self, inputs):
        """A Transformer LM's cached attention takes at most DECODE_MAX_LEN positions, and a prefix can be T' long."""
        if self.lm_fusion and self.lm.model_type == 'transformer_lm':
            T2 = self.model.frontend.output_length(inputs.shape[1])
            if T2 > ops.DECODE_MAX_LEN:
                raise ValueError(f"CTCRecognizer: lm_fusion with a Transformer LM takes at most {ops.DECODE_MAX_LEN} encoder "
                                 f"frames (a prefix can be T' tokens long), got T' = {T2}")

    def _fused_search(self, B, T2, K, device):
        """The fused search of one geometry; the most recent few are kept (each owns its buffers and its graph)."""
        key = (B, T2, K, device.index, self.lm, float(self.lm_weight), float(self.beta))   # launch arguments a graph bakes in
        return lru_get(self._searches, key, 2, lambda: CTCFusedSearch(
            self.lm, B, self.beam_width, T2, K, device, self.lm_weight, self.beta, self.model.assistor.blank, self.use_graph))

    def recognize_ids(self, inputs, inputs_mask):
        """-> (ids i64 [B, nbest, T'] best first, 0 after each hypothesis' end; lengths i32 [B, nbest]; scores f32 [B, nbest]),
        on the device.  nbest is 1 in greedy mode (score: the best path's log-prob) and beam_width in beam mode (score:
        the prefix's log-probability over all its alignments)."""
        self._check_frames(inputs)
        with torch.no_grad():
            return self._decode(*self.model.logits_bf16(inputs, inputs_mask))

    def _decode(self, logits, lengths, B, T2):
        if self.lm_fusion:
            V = self.model.vocab_size
            K = min(CTC_CUTOFF_TOP_N, V)
            lp, tok = ops.ctc_frame_topk(logits, B, T2, V, lengths, K)
            return self._fused_search(B, T2, K, logits.device).run(lp, tok, lengths)
        ids, n, sc = ctc_decode(logits, lengths, B, T2, self.model.vocab_size, self.model.assistor.blank, self.mode,
                                self.beam_width)
        if not self.apply_lm_rescoring:
            return ids, n, sc
        return rescore_nbest(ids, sc, [lambda x, y, K, Lp: lm_token_logprob(self.lm, x, y)], self.rescore_weight,
                             self.beam_width, width=T2, pad=PAD, lengths=n)

    def recognize_spans(self, inputs, inputs_mask):
        """recognize_ids, plus where each token of the 1-best lies: the 1-best is force-aligned (otb_ctc_align) against the
        same logits, so the front end and encoder run once.  -> (ids, lengths, scores as recognize_ids; spans i32
        [B, min(T', 1023), 2] [start, end) in encoder frames of the 1-best's tokens, -1 past its length, and -1 throughout
        for a 1-best longer than the aligner's 1023 tokens), on the device.
        model.encoder_frames_to_input converts the spans to input frames or seconds."""
        self._check_frames(inputs)
        with torch.no_grad():
            logits, lengths, B, T2 = self.model.logits_bf16(inputs, inputs_mask)
            ids, n, sc = self._decode(logits, lengths, B, T2)
            best = ids[:, 0, :min(T2, ops.CTC_ALIGN_MAX_TOKENS)]
            _, _, spans, _ = ctc_align_logits(logits, lengths, B, T2, self.model.vocab_size, best, n[:, 0], self.model.assistor.blank)
            return ids, n, sc, spans

    def recognize(self, inputs, inputs_mask):
        """recognize/ctc.py:27-36: translate() of the 1-best token lists (the id lists when idx2unit is None)."""
        ids, n, _ = self.recognize_ids(inputs, inputs_mask)
        best = [row[:k] for row, k in zip(ids[:, 0].cpu().tolist(), n[:, 0].cpu().tolist())]
        return best if self.idx2unit is None else self.translate(best)


class _TransducerSearch(FusedLMRows):
    """A transducer search of one geometry (B utterances, T' frames, N rows) over the model's current operands: the encoder
    projection Ep, the prediction network, the LM-fusion set-up, and the loop of blocks of STEPS steps.  A block is a
    graphs.CapturedStep keyed on the model's and the fused LM's weight packs, so new weights recapture it in place; the
    host reads the live-row counter once per block.  A subclass allocates its own buffers (self.out: what run returns,
    self.active: the live-row counter) and writes start_rows (its state before the first step) and _step."""

    STEPS = 16          # search steps per graph replay: the host reads the live-row counter once per replay

    def __init__(self, model, B, T2, N, k, max_len, device, use_graph, lm, lm_weight, beta):
        self.model, self.B, self.T2, self.max_len = model, B, T2, max_len
        D, H, L = model.joint.inner_size, model.decoder.hidden_size, model.decoder.num_layers
        f32, i32 = dict(dtype=torch.float32, device=device), dict(dtype=torch.int32, device=device)
        self.ep = torch.empty(B * T2, D, dtype=ops.BF16, device=device)
        self.ep_cur, self.pp = (torch.empty(N, D, dtype=ops.BF16, device=device) for _ in range(2))
        self.h, self.c = (torch.empty(L, N, H, **f32) for _ in range(2))
        self.logp = torch.empty(N, model.joint.ld_logits, **f32)
        self.val = torch.empty(N, k, **f32)
        self.idx = torch.empty(N, k, **i32)
        self.tok = torch.zeros(N, dtype=torch.long, device=device)
        self.t_len = torch.zeros(B, **i32)
        self.bar = torch.zeros(2, **i32)            # the LSTM kernels' grid barrier, owned here: a graph must not allocate one
        self.lm, self.lm_weight, self.beta = lm, float(lm_weight), float(beta)
        self.op = None                              # the model's operands, read by start()
        self.block = CapturedStep(self._steps, self._packs, use_graph)

    def _packs(self):
        return (self.op,) if self.lm is None else (self.op, self.lm._pack.get())

    def _predict(self, hidden):
        """The prediction network one token on from hidden (None: the zero state) for every row's self.tok -> (h, c,
        dec_proj(h))."""
        op = self.op
        x = ops.embedding(self.tok, op['emb'])
        y, h, c, _ = train.lstm_stack_fwd(x, op['layers'], 1, self.tok.numel(), hidden=hidden, barrier=self.bar)
        return h, c, ops.linear(y, op['dec_w'])

    def start(self, mem, lengths):
        """The state before the first step: Ep of the memory, the subclass's rows, every row's prediction network from BLK
        and the zero state, and the LM on <S/E>."""
        self.op = self.model._pack.get()
        enc = self.op['enc']
        ops.linear(mem, enc.w, enc.b, ops.EPI_BIAS, out=self.ep)
        self.t_len.copy_(lengths)
        self.start_rows(lengths)
        self.tok.zero_()
        h, c, pp = self._predict(None)
        self.h.copy_(h)
        self.c.copy_(c)
        self.pp.copy_(pp)
        if self.lm is not None:
            self.start_lm()

    def _steps(self):
        for _ in range(self.STEPS):
            self._step()

    def run(self, mem, lengths):
        self.start(mem, lengths)
        self.steps = 0
        # every step moves each live row one frame on or one label on: T_b + max_len steps end every utterance
        for _ in range(-(-(self.T2 + self.max_len) // self.STEPS)):
            self.block()
            self.steps += self.STEPS
            if int(read_device(self.active)[0]) == 0:
                break
        return tuple(t.clone() for t in self.out)


class _TransducerGreedy(_TransducerSearch):
    """The greedy transducer search: one row per utterance.  With an LM (shallow fusion, DESIGN.md 4.22) each row also
    carries log p_lm(. | <S/E>, its labels): the LM runs on every row's arg-max after the step, and the rows that emitted
    keep it."""

    def __init__(self, model, B, T2, max_len, max_sym, device, use_graph, lm=None, lm_weight=0.0, beta=0.0):
        super().__init__(model, B, T2, B, 1, max_len, device, use_graph, lm, lm_weight, beta)
        self.max_sym = max_sym
        i32 = dict(dtype=torch.int32, device=device)
        self.frame, self.n_sym, self.n_out = (torch.zeros(B, **i32) for _ in range(3))
        self.ids = torch.zeros(B, max_len, **i32)
        self.score = torch.zeros(B, dtype=torch.float32, device=device)
        self.out = (self.ids, self.n_out, self.score)
        self.active = torch.zeros(1, **i32)
        if lm is not None:
            # one LM row per utterance; the Transformer LM's cache is linear, position p of utterance b at row b L + p
            L = max_len + 1
            row = torch.arange(B, device=device)
            self._init_lm(lm, B, L, B * L, row * L, torch.zeros_like(row), device)
            if self.anc is not None:
                self.anc.copy_(row[:, None] * L + torch.arange(L, device=device))

    def start_rows(self, lengths):
        for t in (self.frame, self.n_sym, self.n_out, self.ids, self.score):
            t.zero_()
        self.active.copy_((lengths > 0).sum().view(1))
        self.ep_cur.copy_(self.ep.view(self.B, self.T2, -1)[:, 0])

    def _step(self):
        op, m = self.op, self.model
        hj = ops.rnnt_joint(self.ep_cur, self.pp, self.B, 1, 1)
        logits = ops.linear(hj, op['out_w'], op['out_b'], ops.EPI_BIAS, out_f32=True, n_out=m.joint.ld_logits)
        if self.lm is None:
            ops.logsoftmax_topk(logits, m.vocab_size, 1, out_val=self.val, out_idx=self.idx, out_logp=self.logp)
        else:
            _fused_topk(self, logits, m.vocab_size, 1)
        self.tok.copy_(self.idx.view(-1))
        h, c, pp = self._predict((self.h, self.c))          # every row's next state, kept only where a label is emitted
        fused = self.lm is not None
        ops.rnnt_greedy_step(self.idx, self.logp, h, c, pp, self.h, self.c, self.pp, self.ep, self.T2, self.ep_cur,
                             self.t_len, self.frame, self.n_sym, self.n_out, self.ids, self.max_sym, self.score, self.active,
                             val=self.val if fused else None, emit=self.ext if fused else None,
                             lm_pos=self.pos if fused else None)
        if fused:
            self.follow(None)                               # the LM on every row's arg-max, kept where it was emitted


class _TransducerALSD(_TransducerSearch):
    """The ALSD beam search (K slots per utterance, an n-best of W, max_len labels): its buffers and the node table.  Every
    array is at B*K slot rows; the step is rnnt_joint -> output layer -> logsoftmax_topk -> otb_rnnt_beam_step ->
    otb_rnnt_beam_gather -> the prediction network one token on -> otb_rnnt_beam_commit.  With an LM (shallow fusion,
    DESIGN.md 4.22) each slot also carries log p_lm(. | <S/E>, its labels), following its parent slot and advanced by the
    LM where it took a label; the Transformer LM's K/V are stored once per node of the node table, [blocks, B n_cap, d],
    node 0 the <S/E>."""

    def __init__(self, model, B, T2, K, W, max_len, device, use_graph, lm=None, lm_weight=0.0, beta=0.0):
        BK = B * K
        self.K, self.k1 = K, min(K + 1, model.vocab_size)
        super().__init__(model, B, T2, BK, self.k1, max_len, device, use_graph, lm, lm_weight, beta)
        D, H, L = model.joint.inner_size, model.decoder.hidden_size, model.decoder.num_layers
        f32, i32 = dict(dtype=torch.float32, device=device), dict(dtype=torch.int32, device=device)
        self.ppg = torch.empty(BK, D, dtype=ops.BF16, device=device)
        self.hg, self.cg = (torch.empty(L, BK, H, **f32) for _ in range(2))
        n_cap = K * (T2 + max_len) + 1                  # the root and at most K new nodes per step, T_b + max_len steps
        if lm is not None:
            row = torch.arange(BK, device=device)
            self._init_lm(lm, BK, max_len + 1, B * n_cap, (row // K) * n_cap, torch.where(row % K == 0, 0, -1), device)
            self.lm_out = dict(src=self.src, ext=self.ext, anc=self.anc, anc_tmp=self.anc_tmp, pos=self.pos)
        # tok: the label each slot took, read by the prediction network and the LM
        self.state = dict(score=torch.empty(BK, **f32), u=torch.empty(BK, **i32), frame=torch.empty(BK, **i32),
                          node=torch.empty(BK, **i32), par=torch.empty(BK, **i32), tok=self.tok,
                          node_par=torch.zeros(B, n_cap, **i32), node_tok=torch.zeros(B, n_cap, **i32),
                          n_nodes=torch.empty(B, **i32), f_score=torch.empty(B, W, **f32), f_node=torch.empty(B, W, **i32),
                          f_u=torch.empty(B, W, **i32), f_n=torch.empty(B, **i32), done=torch.empty(B, **i32),
                          active=torch.empty(1, **i32))
        self.active = self.state['active']
        self.out = (torch.zeros(B, W, max_len, **i32), torch.zeros(B, W, **i32), torch.empty(B, W, **f32))

    def step_phases(self):
        """One search step as its seven phases, in order (tools/transducer_beam.py times each)."""
        op, m, s = self.op, self.model, self.state
        box = {}

        def joint():
            box['hj'] = ops.rnnt_joint(self.ep_cur, self.pp, self.B * self.K, 1, 1)

        def output_layer():
            box['logits'] = ops.linear(box['hj'], op['out_w'], op['out_b'], ops.EPI_BIAS, out_f32=True, n_out=m.joint.ld_logits)

        def topk():
            if self.lm is None:
                ops.logsoftmax_topk(box['logits'], m.vocab_size, self.k1, out_val=self.val, out_idx=self.idx,
                                    out_logp=self.logp)
            else:
                _fused_topk(self, box['logits'], m.vocab_size, self.k1)

        def beam_step():
            if self.lm is None:
                ops.rnnt_beam_step(self.logp, self.val, self.idx, m.vocab_size, self.T2, self.t_len, s, self.out)
            else:
                ops.rnnt_beam_step(self.logp, self.val, self.idx, m.vocab_size, self.T2, self.t_len, s, self.out, self.beta,
                                   self.lm_out)

        def gather():
            ops.rnnt_beam_gather(s['par'], s['frame'], self.K, self.h, self.c, self.pp, self.ep, self.T2, self.hg, self.cg,
                                 self.ppg, self.ep_cur)

        def predictor():            # every slot's next state, kept only where it took a label
            box['new'] = self._predict((self.hg, self.cg))

        def commit():
            ops.rnnt_beam_commit(s['tok'], self.hg, self.cg, self.ppg, *box['new'], self.h, self.c, self.pp)

        def lm():                   # every slot's LM rows from its parent, the LM one token on where it took a label
            self.follow(self.src)
        return [joint, output_layer, topk, beam_step, gather, predictor, commit] + ([lm] if self.lm is not None else [])

    def _step(self):
        for phase in self.step_phases():
            phase()

    def start_rows(self, lengths):
        """One live slot per utterance with a frame, the empty sequence at frame 0."""
        B, T2, K, s = self.B, self.T2, self.K, self.state
        s['score'].fill_(float('-inf'))
        s['score'].view(B, K)[:, 0].masked_fill_(lengths > 0, 0.0)
        for k in ('u', 'frame', 'node', 'par', 'f_n', 'done'):
            s[k].zero_()
        s['n_nodes'].fill_(1)
        s['active'].fill_(B)                    # an utterance without frames ends at the first step
        for t in self.out[:2]:
            t.zero_()
        self.out[2].fill_(float('-inf'))
        self.ep_cur.view(B, K, -1).copy_(self.ep.view(B, T2, -1)[:, :1])


def _fused_topk(search, logits, V, k):
    """logsoftmax_topk with the transducer's fusion: labels valued lp + lm_weight * lm + beta, blank (column 0) its plain
    log-prob, out_logp the plain log-probs.  At lm_weight 0 the LM rows are not read (0 * -inf would be NaN)."""
    ops.logsoftmax_topk(logits, V, k, search.lm_rows if search.lm_weight != 0 else None, search.lm_weight, out_val=search.val,
                        out_idx=search.idx, out_logp=search.logp, lm_beta=search.beta, lm_exempt=0)


class TransducerRecognizer(Recognizer):
    """Search of a TransducerModel (DESIGN.md 4.22), batched on the device.

    mode='greedy': at each step every live utterance takes the arg-max of the joint's log-probs at its current frame and
    predictor state (ties to the lower id): a label is emitted and the prediction network advances, at most
    max_symbols_per_frame times per frame and max_len tokens in all (after which only blank is taken); blank moves to the
    next frame.  The score is the sum of the chosen log-probs, blanks included.  All decisions run in one kernel per step
    (otb_rnnt_greedy_step).  beam_width is ignored and nbest must be 1.

    mode='alsd': alignment-length synchronous beam search (Saon et al. 2020) with beam_width K (1..15) hypotheses per
    utterance and an n-best of nbest (1..K).  Every hypothesis takes one lattice step per search step: blank (one frame on)
    or one of its K best labels (while it has fewer than max_len); hypotheses with the same labels at the same step are
    merged by log-adding their scores, so a score sums every alignment of its labels the beam kept.  A hypothesis that takes
    blank on its last frame is a final; the n-best holds the nbest best finals, and an utterance ends when no hypothesis is
    live or the live ones together can no longer beat the n-best's worst.  max_symbols_per_frame does not apply: ALSD
    bounds labels by max_len alone.  One kernel per step makes every decision (otb_rnnt_beam_step).

    lm (the Transformer or the recurrent LM of opentransformer_b200.lm), without apply_lm_rescoring: shallow fusion in
    either mode (DESIGN.md 4.22).  A label k taken by a hypothesis with labels y adds lp(k) + lm_weight *
    log p_lm(k | <S/E>, y) + beta, blank adds lp(blank) alone; the labels a hypothesis offers (greedy: its arg-max) are
    chosen by that fused value, and the scores are the fused totals.  No end-of-sentence term is added.

    apply_lm_rescoring (ALSD only): the LM is not fused; the search keeps beam_width finals, which are re-ranked by
    s + rescore_weight * log P_lm(y <S/E>) (DESIGN.md 4.10), and the nbest best are returned.

    Both modes capture a block of steps in a CUDA graph (use_graph=False: launched one by one) and replay it until a device
    counter shows every utterance ended; new weights, the model's or the fused LM's, capture it again.  The default and modified beam searches and n-gram scoring are not implemented."""

    def __init__(self, model, idx2unit=None, max_symbols_per_frame=5, max_len=1023, ngpu=1, use_graph=True, lm=None,
                 ngram_lm=None, mode='greedy', beam_width=5, nbest=1, lm_weight=0.1, beta=0.0, apply_lm_rescoring=False,
                 rescore_weight=1.0):
        if mode == 'beam':
            raise NotImplementedError("TransducerRecognizer: the default (Graves) beam search is not implemented; "
                                      "mode='alsd' is the transducer beam search")
        if mode not in ('greedy', 'alsd'):
            raise NotImplementedError(f"TransducerRecognizer: mode must be 'greedy' or 'alsd', got {mode!r}")
        if apply_lm_rescoring:
            if mode != 'alsd':
                raise ValueError("TransducerRecognizer: apply_lm_rescoring re-ranks an n-best; greedy search has one "
                                 "hypothesis, use mode='alsd'")
            check_lm_rescoring('TransducerRecognizer', lm, model.vocab_size)
        elif lm is not None:
            check_lm_fusion('TransducerRecognizer', lm, model.vocab_size)
            if not lm_weight >= 0:
                raise ValueError(f'TransducerRecognizer: lm_weight must be >= 0, got {lm_weight}: the early end of the '
                                 'ALSD search needs the LM term to be at most 0')
            if lm.model_type == 'transformer_lm' and max_len + 1 > ops.DECODE_MAX_LEN:
                raise ValueError(f"TransducerRecognizer: the Transformer LM's cached attention holds {ops.DECODE_MAX_LEN} "
                                 f'positions, <S/E> and max_len = {max_len} labels need {max_len + 1}')
        if ngram_lm is not None:
            raise NotImplementedError('TransducerRecognizer: n-gram LM scoring (KenLM) is not implemented; use ngram_lm=None')
        if not 1 <= max_len <= ops.RNNT_MAX_LABELS:
            raise ValueError(f'TransducerRecognizer: max_len must be in [1, {ops.RNNT_MAX_LABELS}], got {max_len}')
        if max_symbols_per_frame < 1:
            raise ValueError(f'TransducerRecognizer: max_symbols_per_frame must be >= 1, got {max_symbols_per_frame}')
        if mode == 'alsd':
            if not 1 <= beam_width <= ops.RNNT_BEAM_MAX:
                raise ValueError(f'TransducerRecognizer: beam_width must be in [1, {ops.RNNT_BEAM_MAX}], got {beam_width}')
            if not 1 <= nbest <= beam_width:
                raise ValueError(f'TransducerRecognizer: nbest must be in [1, beam_width = {beam_width}], got {nbest}')
        elif nbest != 1:
            raise ValueError(f"TransducerRecognizer: greedy search has one hypothesis, got nbest={nbest}; use mode='alsd'")
        super().__init__(model, idx2unit, lm, lm_weight, ngpu)
        self.max_len, self.max_symbols_per_frame, self.use_graph = int(max_len), int(max_symbols_per_frame), bool(use_graph)
        self.mode, self.beam_width, self.nbest = mode, int(beam_width), int(nbest)
        self.lm_weight, self.beta = float(lm_weight), float(beta)
        self.apply_lm_rescoring, self.rescore_weight = bool(apply_lm_rescoring), float(rescore_weight)
        self._search = None

    def recognize_ids(self, inputs, inputs_mask):
        """greedy: -> (ids i32 [B, max_len], 0 after each utterance's tokens; lengths i32 [B]; scores f32 [B]);
        alsd: -> (ids i32 [B, nbest, max_len]; lengths i32 [B, nbest]; scores f32 [B, nbest]), best first, entries past the
        finals found with length 0 and score -inf; on the device."""
        with torch.no_grad():
            mem, lengths, B, T2 = self.model.encode_bf16(inputs, inputs_mask)
            s = self._search
            # a search owns the buffers of one geometry; new weights (the model's or the fused LM's) recapture its graph
            if s is None or (s.B, s.T2, s.ep.device) != (B, T2, mem.device):
                fusion = dict(lm=None if self.apply_lm_rescoring else self.lm, lm_weight=self.lm_weight, beta=self.beta)
                if self.mode == 'alsd':
                    W = self.beam_width if self.apply_lm_rescoring else self.nbest
                    s = _TransducerALSD(self.model, B, T2, self.beam_width, W, self.max_len, mem.device, self.use_graph,
                                        **fusion)
                else:
                    s = _TransducerGreedy(self.model, B, T2, self.max_len, self.max_symbols_per_frame, mem.device,
                                          self.use_graph, **fusion)
                self._search = s
            self.model.decoder._check_device(mem.device)
            out = s.run(mem, lengths)
            if not self.apply_lm_rescoring:
                return out
            ids, n, sc = out
            ids, n, sc = rescore_nbest(ids, sc, [lambda x, y, K, Lp: lm_token_logprob(self.lm, x, y)], self.rescore_weight,
                                       self.nbest, width=self.max_len, pad=PAD, lengths=n)
            return ids.int(), n, sc

    def recognize(self, inputs, inputs_mask):
        """greedy: translate() of the 1-best token lists (the id lists when idx2unit is None), as CTCRecognizer.recognize.
        alsd: (nbest_translate(ids), scores), as SpeechToTextRecognizer.recognize: with idx2unit, each utterance's n-best
        strings (an entry without a final is ''); without, the id tensor [B, nbest, max_len]."""
        ids, n, sc = self.recognize_ids(inputs, inputs_mask)
        if self.mode == 'alsd':
            if self.idx2unit is None:
                return self.nbest_translate(ids), sc
            # the EOS that ends nbest_translate's rows: ids past each length are padding (0), which has no unit
            cut = torch.arange(ids.shape[2], device=ids.device) >= n.unsqueeze(2)
            return self.nbest_translate(ids.masked_fill(cut, EOS).long()), sc
        best = [row[:k] for row, k in zip(ids.cpu().tolist(), n.cpu().tolist())]
        return best if self.idx2unit is None else self.translate(best)


def build_recognizer(model_type, model, lm, args, idx2unit):
    """otrans/recognize/__init__.py:5-21."""
    if model_type == 'speech2text':
        return SpeechToTextRecognizer(
            model=model, lm=lm, lm_weight=args.lm_weight, ctc_weight=args.ctc_weight, beam_width=args.beam_width,
            nbest=args.nbest, max_len=args.max_len, idx2unit=idx2unit, penalty=args.penalty, lamda=args.lamda,
            ngpu=args.ngpu, ctc_candidates=getattr(args, 'ctc_candidates', None),
            apply_rescoring=getattr(args, 'apply_rescoring', False),
            apply_lm_rescoring=getattr(args, 'apply_lm_rescoring', False), rescore_weight=getattr(args, 'rescore_weight', 1.0),
            apply_ctc_rescoring=getattr(args, 'apply_ctc_rescoring', False))
    if model_type == 'ctc':
        if getattr(args, 'apply_rescoring', False):
            raise ValueError('build_recognizer: apply_rescoring re-scores with the attention decoder, and a CTC model has none')
        if getattr(args, 'apply_ctc_rescoring', False):
            raise ValueError('build_recognizer: apply_ctc_rescoring re-scores the n-best of the attention beam search, and a '
                             'CTC model has none')
        return CTCRecognizer(
            model=model, lm=lm, lm_weight=args.lm_weight, ngram_lm=args.ngram_lm, beam_width=args.beam_width,
            idx2unit=idx2unit, ngpu=args.ngpu, mode=args.mode, alpha=args.alpha, beta=args.beta,
            apply_lm_rescoring=getattr(args, 'apply_lm_rescoring', False), rescore_weight=getattr(args, 'rescore_weight', 1.0),
            lm_fusion=getattr(args, 'lm_fusion', False))
    if model_type == 'transducer':
        return TransducerRecognizer(model=model, idx2unit=idx2unit, max_len=getattr(args, 'max_len', 1023), ngpu=args.ngpu,
                                    lm=lm, ngram_lm=getattr(args, 'ngram_lm', None), mode=getattr(args, 'mode', 'greedy'),
                                    max_symbols_per_frame=getattr(args, 'max_symbols_per_frame', 5),
                                    beam_width=getattr(args, 'beam_width', 5), nbest=getattr(args, 'nbest', 1),
                                    lm_weight=getattr(args, 'lm_weight', 0.1), beta=getattr(args, 'beta', 0.0),
                                    apply_lm_rescoring=getattr(args, 'apply_lm_rescoring', False),
                                    rescore_weight=getattr(args, 'rescore_weight', 1.0))
    raise NotImplementedError(model_type)
