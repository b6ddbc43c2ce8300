"""Regenerate tests/golden/live_ref_ctc.pt from the reference's OWN modules (byte-compiled into oracle/_ref by
oracle/build_ref.py), on the CPU:

  train       End2EndModel['ctc'] in train() with residual_dropout 0, once with a Transformer encoder and once with a
              Conformer encoder (d_model 128, 2 heads: 64 wide, kernel 5): `loss, _ = model(inputs, targets);
              loss.backward()` on a ragged, PAD-padded batch whose label counts differ.  Stored: the loss, every parameter
              gradient (None where .grad stayed None; a fixed quarter of each tensor larger than 4096 elements,
              tests/test_transformer_lm_ref.sample) and the BatchNorm running statistics after the forward.  Weights are
              stored as key shapes + seed (tests/test_head_dim_96.synth_state_dict).
  greedy      CTCRecognizer(mode='greedy', ngpu=0).recognize_greedy driven by a stub model whose inference returns stored
              log-probs: its id lists.  The utterances hold repeats split by blank, runs of one token, an all-blank
              utterance and a length-1 utterance.
  baseline    the key names and shapes of a CTC model with the transformer_baseline.yaml front end and encoder.

    python oracle/build_ref.py && python tests/golden/make_live_ref_ctc.py     # needs the reference tree
"""
import copy
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.test_head_dim_96 import synth_state_dict  # noqa: E402
from tests.test_transformer_lm_ref import sample  # noqa: E402

SEED = 512
V = 30
FRONTEND = dict(input_size=20, output_size=128, in_channel=1, mid_channel=4, out_channel=8, kernel_size=[[3, 3], [3, 3]],
                stride=[2, 2], dropout=0.0, act_func_type='relu', front_end_layer_norm=False)
ENCODERS = {
    'transformer': dict(d_model=128, n_heads=2, d_ff=96, n_blocks=2, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                        residual_dropout=0.0, normalize_before=False, concat_after=False, activation='glu',
                        relative_positional=False),
    'conformer': dict(d_model=128, d_ff=96, cov_kernel_size=5, n_heads=2, nblocks=2, pos_dropout=0.0, slf_attn_dropout=0.0,
                      ffn_dropout=0.0, residual_dropout=0.0, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5,
                      conv_bias=True, activation='glu', positional_encoding=True, relative_positional=True),
}


def params(encoder_type):
    return {'type': 'ctc', 'frontend_type': 'conv', 'encoder_type': encoder_type, 'frontend': copy.deepcopy(FRONTEND),
            'encoder': copy.deepcopy(ENCODERS[encoder_type]), 'encoder_output_size': 128, 'vocab_size': V}


def baseline_params():
    """transformer_baseline.yaml's front end and encoder under a CTC head (vocab 4234)."""
    return {'type': 'ctc', 'frontend_type': 'conv', 'encoder_type': 'transformer',
            'frontend': dict(input_size=80, output_size=256, in_channel=1, mid_channel=64, out_channel=128,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=256, n_heads=4, d_ff=2048, n_blocks=12, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.1, normalize_before=False, concat_after=False,
                            activation='glu', relative_positional=False),
            'encoder_output_size': 256, 'vocab_size': 4234}


def batch():
    """Ragged inputs; truth = BOS, labels, EOS, PAD* with 6, 3 and 4 labels."""
    g = torch.Generator().manual_seed(23)
    B, T, L = 3, 70, 8
    lens = torch.tensor([70, 55, 41])
    mask = torch.arange(T)[None] < lens[:, None]
    x = torch.randn(B, T, 20, generator=g) * mask.unsqueeze(2)
    tgt = torch.randint(2, V, (B, L), generator=g)
    tgt[:, 0] = 1
    tgt[0, 7] = 1
    tgt[1, 4:] = torch.tensor([1, 0, 0, 0])
    tgt[2, 5:] = torch.tensor([1, 0, 0])
    tgt[2, 2] = tgt[2, 3]                     # a doubled label: the alignment needs a blank between them
    return x, mask, tgt, (tgt[:, 1:] != 0).sum(1)


def train_case(encoder_type):
    from otrans.model import End2EndModel
    p = params(encoder_type)
    ref = End2EndModel['ctc'](p)
    shapes = {k: (tuple(v.shape), str(v.dtype).replace('torch.', '')) for k, v in ref.state_dict().items()}
    ref.load_state_dict(synth_state_dict(shapes, SEED), strict=True)
    ref.train()
    x, mask, tgt, tlen = batch()
    loss, aux = ref({'inputs': x, 'mask': mask}, {'targets': tgt, 'targets_length': tlen})
    assert aux is None
    loss.backward()
    grads = {n: (sample(q.grad) if q.grad is not None else None) for n, q in ref.named_parameters()}
    stats = {n: b.detach().clone() for n, b in ref.named_buffers() if 'running_' in n or 'num_batches' in n}
    return {'params': p, 'sd_shapes': shapes, 'sd_seed': SEED, 'x': x, 'mask': mask, 'tgt': tgt, 'tlen': tlen,
            'loss_ref': loss.detach(), 'g_ref': grads, 'stats_ref': stats}


def greedy_log_probs():
    """[B, T, V] log-probs whose best tokens hold the patterns the collapse must get right, and their lengths."""
    g = torch.Generator().manual_seed(29)
    B, T, Vg = 5, 12, 7
    best = torch.tensor([
        [3, 3, 0, 3, 5, 5, 5, 0, 0, 2, 2, 4],       # a repeat split by blank, then a run of one token
        [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0],       # all blank
        [6, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0],       # length 1
        [1, 1, 2, 0, 2, 2, 0, 0, 1, 3, 0, 3],       # token 1 (<S/E>) among the labels, repeats around blanks
        [4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4, 4],       # one run over the whole utterance
    ])
    lengths = torch.tensor([12, 9, 1, 12, 7])
    lp = torch.randn(B, T, Vg, generator=g)
    lp.scatter_(2, best.unsqueeze(2), 4.0)
    return torch.log_softmax(lp, dim=-1), lengths


class _StubModel(torch.nn.Module):
    def __init__(self, lp, lengths):
        super().__init__()
        self.lp, self.lengths = lp, lengths

    def inference(self, inputs, inputs_length):
        return self.lp, self.lengths


def greedy_case():
    from otrans.recognize.ctc import CTCRecognizer
    lp, lengths = greedy_log_probs()
    rec = CTCRecognizer(_StubModel(lp, lengths), mode='greedy', ngpu=0, beam_width=1, idx2unit={i: str(i) for i in range(7)})
    return {'lp': lp, 'lengths': lengths, 'ids_ref': rec.recognize_greedy(None, None)}


def baseline_case():
    from otrans.model import End2EndModel
    ref = End2EndModel['ctc'](baseline_params())
    return {'params': baseline_params(), 'shapes': {k: tuple(v.shape) for k, v in ref.state_dict().items()}}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    torch.save({'train': {e: train_case(e) for e in ENCODERS}, 'greedy': greedy_case(), 'baseline': baseline_case()},
               os.path.join(HERE, 'live_ref_ctc.pt'))
