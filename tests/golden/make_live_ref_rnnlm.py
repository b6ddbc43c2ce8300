"""Regenerate the recurrent-LM fixture from the reference's OWN RecurrentLanguageModel (model/lm.py:31-90, byte-compiled into
oracle/_ref by oracle/build_ref.py):

  live_ref_rnnlm.pt   for a tied and an untied model (vocab 40, hidden 64, 2 layers, dropout 0.0) on deterministic weights
                      (tests/test_rnnlm_ref.synth_state_dict: only the key shapes and the seed are stored): PAD-padded inputs
                      and targets, predict() with the zero state and with the hidden state carried over two calls, the loss
                      of forward() in train() and every parameter gradient after loss.backward(); and {state_dict key:
                      shape} of the full rnnlm.yaml model (no weights)

    python oracle/build_ref.py && python tests/golden/make_live_ref_rnnlm.py     # needs the reference tree
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_ref  # noqa: E402
from tests.test_rnnlm_ref import RNNLM_YAML, small_params, small_batch, synth_state_dict  # noqa: E402


def case(tied, seed):
    from otrans.model.lm import RecurrentLanguageModel
    params = small_params(tied)
    ref = RecurrentLanguageModel(params)
    shapes = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    ref.load_state_dict(synth_state_dict(shapes, seed, tied), strict=True)
    inputs, targets = small_batch()
    ref.eval()
    with torch.no_grad():
        logp, (h, c) = ref.predict(inputs)
        lp1, hid1 = ref.predict(inputs[:, :4])
        lp2, (h2, c2) = ref.predict(inputs[:, 4:], hid1)
    ref.train()
    loss, _ = ref({'inputs': inputs}, {'targets': targets})
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in ref.named_parameters()}
    return {'params': params, 'sd_shapes': shapes, 'sd_seed': seed, 'inputs': inputs, 'targets': targets,
            'log_probs': logp, 'h_n': h, 'c_n': c, 'carried_log_probs': torch.cat([lp1, lp2], 1), 'carried_h_n': h2,
            'carried_c_n': c2, 'loss': loss.detach(), 'grads': grads}


def rnnlm_yaml_keys():
    from otrans.model.lm import RecurrentLanguageModel
    return {k: tuple(v.shape) for k, v in RecurrentLanguageModel(RNNLM_YAML).state_dict().items()}


if __name__ == '__main__':
    if build_ref.load() is None:
        raise SystemExit('oracle/_ref is missing: run oracle/build_ref.py where the reference tree exists')
    torch.save({'tied': case(True, 41), 'untied': case(False, 42), 'rnnlm_yaml_keys': rnnlm_yaml_keys()},
               os.path.join(HERE, 'live_ref_rnnlm.pt'))
    print('wrote live_ref_rnnlm.pt to', HERE)
