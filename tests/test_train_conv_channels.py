"""The training path takes conv front ends up to 256 (padded) mid channels, which is what the conv1 weight gradient kernel
handles (one channel per thread).  A wider front end must be refused up front, without a GPU, instead of failing in the
middle of the backward."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _params(mid_channel):
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
            'frontend': dict(input_size=80, output_size=256, in_channel=1, mid_channel=mid_channel, out_channel=32,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=256, n_heads=4, d_ff=256, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                            residual_dropout=0.1, normalize_before=False, concat_after=False, activation='glu',
                            relative_positional=False),
            'decoder': dict(vocab_size=40, d_model=256, n_heads=4, d_ff=256, memory_dim=256, n_blocks=1, pos_dropout=0.0,
                            slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.1, activation='glu',
                            normalize_before=False, concat_after=False, share_embedding=True),
            'ctc_weight': 0.0, 'smoothing': 0.1}


@pytest.mark.parametrize('mid_channel', [257, 320])
def test_training_refuses_more_than_256_mid_channels(mid_channel):
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.train import TrainPack
    m = SpeechToText(_params(mid_channel))
    with pytest.raises(NotImplementedError, match=f'mid_channel {mid_channel} pads to'):
        TrainPack(m)


@pytest.mark.parametrize('mid_channel', [64, 150, 192, 256])
def test_training_accepts_up_to_256_mid_channels(mid_channel):
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.train import TrainPack
    pk = TrainPack(SpeechToText(_params(mid_channel)))
    assert pk.fe['C1p'] == (mid_channel + 63) // 64 * 64 <= 256
