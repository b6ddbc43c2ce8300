"""96-wide attention heads (d_model 384 / 4 heads, the shipped Conformer configuration) without a GPU:
  * the oracle port reproduces what the reference's own modules computed on a small d_k = 96 model
    (tests/golden/live_ref_dk96.pt, written by tests/golden/make_live_ref_dk96.py: Conformer rel-pos encoder + Transformer
    decoder, d_model 192, 2 heads);
  * the drop-in model builds from the conformer_baseline model dict, with the reference's state_dict key names and shapes
    (tests/golden/live_ref_conformer_baseline_keys.pt);
  * head widths other than 64 and 96 are refused, and so is training with 96-wide heads (the attention backward is 64-wide)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import beam_search as obs      # noqa: E402
from oracle import speech_model as om      # noqa: E402

# `model:` section of the reference's egs/aishell/conf/conformer_baseline.yaml
CONFORMER_BASELINE = {
    'type': 'speech2text', 'frontend_type': 'conv',
    'frontend': dict(input_size=80, output_size=384, in_channel=1, mid_channel=256, out_channel=256,
                     kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu', front_end_layer_norm=False),
    'encoder_type': 'conformer',
    'encoder': dict(d_model=384, d_ff=768, cov_kernel_size=5, n_heads=4, nblocks=12, pos_dropout=0.0, slf_attn_dropout=0.0,
                    ffn_dropout=0.0, residual_dropout=0.1, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5, conv_bias=True,
                    activation='glu', positional_encoding=True, relative_positional=True),
    'decoder_type': 'transformer',
    'decoder': dict(vocab_size=4234, d_model=384, n_heads=4, d_ff=768, memory_dim=384, n_blocks=6, pos_dropout=0.0,
                    slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.1, activation='glu',
                    normalize_before=False, concat_after=False, share_embedding=True),
    'ctc_weight': 0.0, 'smoothing': 0.1}


def dk96_params():
    """Small model with 96-wide heads: Conformer rel-pos encoder and Transformer decoder, d_model 192, 2 heads, 2 blocks each.
    The output layer is untied: with a random tied embedding the search only ever emits EOS."""
    return {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'conformer', 'decoder_type': 'transformer',
            'frontend': dict(input_size=80, output_size=192, in_channel=1, mid_channel=64, out_channel=16,
                             kernel_size=[[3, 3], [3, 3]], stride=[2, 2], dropout=0.0, act_func_type='relu',
                             front_end_layer_norm=False),
            'encoder': dict(d_model=192, d_ff=48, cov_kernel_size=5, n_heads=2, nblocks=2, pos_dropout=0.0, slf_attn_dropout=0.0,
                            ffn_dropout=0.0, residual_dropout=0.0, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5,
                            conv_bias=True, activation='glu', positional_encoding=True, relative_positional=True),
            'decoder': dict(vocab_size=40, d_model=192, n_heads=2, d_ff=48, memory_dim=192, n_blocks=2, pos_dropout=0.0,
                            slf_attn_dropout=0.0, src_attn_dropout=0.0, ffn_dropout=0.0, residual_dropout=0.0,
                            activation='glu', normalize_before=False, concat_after=False, share_embedding=False),
            'ctc_weight': 0.0, 'smoothing': 0.1}


def synth_state_dict(shapes, seed):
    """Deterministic weights for {key: (shape, dtype name)}, drawn in key order from one seeded CPU generator and rounded to
    bf16: the dk96 fixture stores this recipe instead of 1.5 M weights.  Linear / conv weights have the std of PyTorch's
    default init (1 / sqrt(3 fan_in)); LayerNorm and BatchNorm affines, BatchNorm running statistics, biases and the rel-pos
    vectors are non-trivial."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k in sorted(shapes):
        shape, dtype = shapes[k]
        if dtype != 'float32':
            sd[k] = torch.zeros(shape, dtype=getattr(torch, dtype))
            continue
        n = torch.randn(shape, generator=g)
        if k.endswith('running_mean'):
            t = 0.3 * n
        elif k.endswith('running_var'):
            t = 1.0 + 0.5 * torch.rand(shape, generator=g)
        elif k.endswith('posu') or k.endswith('posv'):
            t = 0.3 * n
        elif k.endswith('.bias'):
            t = 0.05 * n
        elif 'norm' in k:                                  # LayerNorm / BatchNorm scale
            t = 1.0 + 0.1 * n
        elif k.endswith('embedding.weight'):
            t = 0.15 * n
        else:                                              # Linear / Conv weight [out, in, ...]
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            t = n / (3.0 * fan_in) ** 0.5
        sd[k] = t.to(torch.bfloat16).float()
    return sd


def load_case(name):
    """live_ref_<name>.pt; the dk96 case carries its state dict as (key shapes, seed) and gets it back from synth_state_dict."""
    c = torch.load(os.path.join(ROOT, 'tests', 'golden', f'live_ref_{name}.pt'), weights_only=False)
    if 'sd_shapes' in c:
        c['sd'] = synth_state_dict(c['sd_shapes'], c['sd_seed'])
    return c


def test_port_equals_live_reference_with_96_wide_heads():
    c = load_case('dk96')
    params, sd, x, mask, beam, max_len = c['params'], c['sd'], c['x'], c['mask'], c['beam'], c['max_len']
    assert params['encoder']['d_model'] // params['encoder']['n_heads'] == 96
    assert params['decoder']['d_model'] // params['decoder']['n_heads'] == 96
    with torch.no_grad():
        mem, mm = om.encode(x, mask, sd, params)
        assert torch.equal(mm, c['mm_ref'])
        torch.testing.assert_close(mem[mm], c['mem_ref'][c['mm_ref']], rtol=1e-4, atol=2e-5)
        nb, ns, _, _ = obs.recognize(x, mask, sd, params, beam=beam, nbest=beam, max_len=max_len, penalty=0.6, lamda=5)
    hyps = c['hyps']
    for b in range(x.shape[0]):
        for r in range(beam):
            port = [int(t) for t in nb[b, r].tolist()]
            port = port[:port.index(1)] if 1 in port else port
            want = [int(t) for t in hyps[b][r].split()] if hyps[b][r] else []
            assert port == want, (b, r, port, want)
    torch.testing.assert_close(ns, c['scores_ref'], rtol=1e-4, atol=1e-4)


def test_conformer_baseline_builds_with_reference_state_dict_names():
    from opentransformer_b200.model import SpeechToText
    want = load_case('conformer_baseline_keys')
    m = SpeechToText(CONFORMER_BASELINE)
    got = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert set(got) == set(want), sorted(set(got) ^ set(want))[:20]
    bad = {k: (got[k], want[k]) for k in got if got[k] != tuple(want[k])}
    assert not bad, bad
    assert got['encoder.blocks.11.mha.qvk_proj.weight'] == (1152, 384)
    assert got['encoder.blocks.0.mha.posu'] == (1, 1, 4, 96)


@pytest.mark.parametrize('part', ['encoder', 'decoder'])
def test_unsupported_head_width_is_refused(part):
    """d_model 320 / 4 heads = 80-wide heads: only 64 and 96 are built."""
    from opentransformer_b200.model import SpeechToText
    params = {k: (dict(v) if isinstance(v, dict) else v) for k, v in CONFORMER_BASELINE.items()}
    params['encoder'].update(nblocks=1)
    params['decoder'].update(n_blocks=1)
    params[part]['d_model'] = 320
    if part == 'encoder':
        params['frontend']['output_size'] = 320
        params['decoder']['memory_dim'] = 320
    with pytest.raises(NotImplementedError, match=r'\(64, 96\)'):
        SpeechToText(params)


def test_unsupported_head_width_is_refused_by_the_modules():
    from opentransformer_b200 import modules
    with pytest.raises(NotImplementedError, match=r'\(64, 96\)'):
        modules.MultiHeadedSelfAttention(4, 320)
    with pytest.raises(NotImplementedError, match=r'\(64, 96\)'):
        modules.MultiHeadedCrossAttention(4, 320, 320)
    with pytest.raises(NotImplementedError, match=r'\(64, 96\)'):
        modules.MultiHeadedSelfAttentionWithRelPos(4, 320)
    with pytest.raises(NotImplementedError):
        modules.MultiHeadedSelfAttention(5, 384)            # d_model not a multiple of n_heads
    modules.MultiHeadedSelfAttention(4, 384)
    modules.MultiHeadedSelfAttentionWithRelPos(2, 192)


def test_training_refuses_96_wide_heads():
    """A d_k = 96 Transformer now constructs for inference; the training path must refuse it before any device work."""
    from opentransformer_b200.model import SpeechToText
    from opentransformer_b200.train import TrainPack
    params = {'type': 'speech2text', 'frontend_type': 'conv', 'encoder_type': 'transformer', 'decoder_type': 'transformer',
              'frontend': dict(CONFORMER_BASELINE['frontend'], mid_channel=64, out_channel=64),
              'encoder': dict(d_model=384, n_heads=4, d_ff=768, n_blocks=1, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                              residual_dropout=0.1, normalize_before=False, concat_after=False, activation='glu',
                              relative_positional=False),
              'decoder': dict(CONFORMER_BASELINE['decoder'], vocab_size=40, n_blocks=1),
              'ctc_weight': 0.0, 'smoothing': 0.1}
    m = SpeechToText(params)
    with pytest.raises(NotImplementedError, match='64-wide attention heads'):
        TrainPack(m)
    params['encoder'].update(d_model=256, n_heads=4)
    params['frontend']['output_size'] = 256
    params['decoder'].update(memory_dim=256)
    with pytest.raises(NotImplementedError, match='the decoder has d_model 384'):
        TrainPack(SpeechToText(params))
