"""Regenerate the Transformer-LM training fixture from the reference's OWN TransformerLanguageModel (model/lm.py:94-171,
byte-compiled into oracle/_ref by oracle/build_ref.py):

  live_ref_transformer_lm.pt   for a tied and an untied model (vocab 40, d_model 128, 2 heads, d_ff 256, 2 blocks,
                               residual_dropout 0.0: torch's dropout masks cannot be replayed) on deterministic weights
                               (tests/test_transformer_lm_ref.synth_state_dict: only the key shapes and the seed are stored):
                               PAD-padded inputs and targets of ragged lengths, the loss of forward() in train() and every
                               parameter gradient after loss.backward() (the elements test_transformer_lm_ref.sample picks:
                               a fixed quarter of each tensor larger than 4096); and {state_dict key: shape} of the full
                               transformer_lm.yaml model (no weights)

    python oracle/build_ref.py && python tests/golden/make_live_ref_transformer_lm.py     # needs the reference tree
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.test_transformer_lm_ref import TLM_YAML, sample, small_params, small_batch, synth_state_dict  # noqa: E402


def case(tied, seed):
    from otrans.model.lm import TransformerLanguageModel
    params = small_params(tied)
    ref = TransformerLanguageModel(params)
    shapes = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    ref.load_state_dict(synth_state_dict(shapes, seed, tied), strict=True)
    inputs, targets = small_batch()
    ref.train()
    loss, _ = ref({'inputs': inputs}, {'targets': targets})
    loss.backward()
    grads = {n: sample(p.grad.detach()) for n, p in ref.named_parameters()}
    return {'params': params, 'sd_shapes': shapes, 'sd_seed': seed, 'inputs': inputs, 'targets': targets,
            'loss': loss.detach(), 'grads': grads}


def transformer_lm_yaml_keys():
    from otrans.model.lm import TransformerLanguageModel
    return {k: tuple(v.shape) for k, v in TransformerLanguageModel(TLM_YAML).state_dict().items()}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    torch.save({'tied': case(True, 51), 'untied': case(False, 52), 'transformer_lm_yaml_keys': transformer_lm_yaml_keys()},
               os.path.join(HERE, 'live_ref_transformer_lm.pt'))
    print('wrote live_ref_transformer_lm.pt to', HERE)
