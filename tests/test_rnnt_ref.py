"""CPU checks of the transducer: the float64 lattice restatement (tests/rnnt_ref.py) against torchaudio's rnnt_loss and
against an enumeration of every alignment; the bf16-policy model restatement against the same loss on its own logits; and
TransducerModel's construction, state-dict keys, checkpoint and the refusals that come before any device work."""
import argparse

import pytest
import torch
import torchaudio.functional as TAF

from opentransformer_b200 import model as M
from opentransformer_b200 import recognize, train
from tests import rnnt_ref


def _lattice(B, T, U, V, seed):
    g = torch.Generator().manual_seed(seed)
    logits = 2.0 * torch.randn(B, T, U + 1, V, generator=g)
    labels = torch.randint(1, V, (B, U), generator=g, dtype=torch.int32)
    return logits, labels


@pytest.mark.parametrize('B,T,U,V,t_len,u_len', [(3, 7, 4, 6, [7, 5, 1], [4, 0, 2]), (2, 12, 9, 30, [12, 3], [9, 9]),
                                                 (1, 1, 0, 5, [1], [0])])
def test_lattice_matches_torchaudio(B, T, U, V, t_len, u_len):
    logits, labels = _lattice(B, T, U, V, seed=B * 100 + T)
    t_len, u_len = torch.tensor(t_len, dtype=torch.int32), torch.tensor(u_len, dtype=torch.int32)
    x = logits.clone().requires_grad_(True)
    want = TAF.rnnt_loss(x, labels, t_len, u_len, blank=0, reduction='mean')
    want.backward()
    x64 = logits.double().requires_grad_(True)
    got = rnnt_ref.batch_loss(x64, labels, t_len, u_len)
    got.backward()
    assert abs(float(got) - float(want)) <= 1e-5 * abs(float(want))
    assert float((x64.grad.float() - x.grad).abs().max()) <= 1e-5


@pytest.mark.parametrize('T,U', [(1, 0), (1, 3), (2, 2), (3, 1), (5, 3), (4, 3)])
def test_lattice_matches_enumeration(T, U):
    logits, labels = _lattice(1, T, U, 7, seed=T * 10 + U)
    lpb, lpy = rnnt_ref.node_logprobs(logits[0].double(), labels[0].long())
    a = rnnt_ref.lattice_nll(lpb, lpy)
    b = rnnt_ref.enumerate_nll(lpb, lpy)
    assert abs(float(a) - float(b)) <= 1e-12 * abs(float(b))


def params(encoder_type='transformer', V=40, layers=1, hidden=64, inner=64, dropout=0.0, rate=0.0):
    fe = dict(input_size=80, output_size=128, in_channel=1, mid_channel=64, out_channel=64, kernel_size=[[3, 3], [3, 3]],
              stride=[2, 2], dropout=0.0, act_func_type='relu', front_end_layer_norm=False)
    if encoder_type == 'transformer':
        enc = dict(d_model=128, n_heads=2, d_ff=256, n_blocks=2, pos_dropout=0.0, slf_attn_dropout=0.0, ffn_dropout=0.0,
                   residual_dropout=rate, normalize_before=False, concat_after=False, activation='glu', relative_positional=False)
    else:
        enc = dict(d_model=128, d_ff=256, cov_kernel_size=5, n_heads=2, nblocks=2, pos_dropout=0.0, slf_attn_dropout=0.0,
                   ffn_dropout=0.0, residual_dropout=rate, conv_dropout=0.0, macaron_style=True, ffn_scale=0.5, conv_bias=True,
                   activation='glu', positional_encoding=True, relative_positional=True)
    return {'type': 'transducer', 'frontend_type': 'conv', 'frontend': fe, 'encoder_type': encoder_type, 'encoder': enc,
            'decoder_type': 'rnn', 'decoder': dict(vocab_size=V, hidden_size=hidden, num_layers=layers, dropout=dropout),
            'joint': {'inner_size': inner}}


def test_model_construction_and_keys():
    model = M.End2EndModel['transducer'](params(layers=2))
    keys = set(model.state_dict())
    for k in ('decoder.embedding.weight', 'decoder.rnn.weight_ih_l0', 'decoder.rnn.weight_hh_l1', 'decoder.rnn.bias_ih_l1',
              'decoder.rnn.bias_hh_l0', 'joint.enc_proj.weight', 'joint.enc_proj.bias', 'joint.dec_proj.weight',
              'joint.output_layer.weight', 'joint.output_layer.bias'):
        assert k in keys, k
    assert 'joint.dec_proj.bias' not in keys
    assert not any(k.startswith('decoder.output') for k in keys)
    assert tuple(model.joint.enc_proj.weight.shape) == (64, 128)
    assert tuple(model.joint.output_layer.weight.shape) == (40, 64)
    assert train.unused_parameters(model) == set()


def test_checkpoint_round_trip(tmp_path):
    a = M.TransducerModel(params())
    path = str(tmp_path / 'model.pt')
    a.save_checkpoint({'model': params()}, path)
    chk = torch.load(path)
    assert set(chk) == {'params', 'frontend', 'encoder', 'decoder', 'joint'}
    torch.manual_seed(5)
    b = M.TransducerModel(params())
    b.load_model(chk)
    for (n, x), (_, y) in zip(a.state_dict().items(), b.state_dict().items()):
        assert torch.equal(x, y), n


def test_refusals_before_device_work():
    with pytest.raises(NotImplementedError, match='multiple of 8'):
        M.TransducerModel(params(hidden=60))
    with pytest.raises(NotImplementedError, match="decoder_type"):
        M.TransducerModel(dict(params(), decoder_type='transformer'))
    model = M.TransducerModel(params())
    x, mask = torch.zeros(2, 40, 80), torch.ones(2, 40, dtype=torch.bool)
    truth = torch.tensor([[1, 5, 6, 1], [1, 7, 1, 0]])
    with pytest.raises(ValueError, match='targets_length'):
        model({'inputs': x, 'mask': mask}, {'targets': truth})
    with pytest.raises(ValueError, match='truth_length'):
        train.transducer_forward_backward(model, x, mask, truth, None)
    # 96-wide heads stay refused with the training path's message
    p = params()
    p['encoder'] = dict(p['encoder'], d_model=192, n_heads=2)
    with pytest.raises(NotImplementedError, match='64-wide attention heads'):
        train.transducer_forward_backward(M.TransducerModel(p), x, mask, truth, torch.tensor([3, 2]))
    with pytest.raises(NotImplementedError, match='attention decoder'):
        train.FusedTrainer(model, mwer_nbest=4)
    with pytest.raises(TypeError, match='truth_length is required'):
        model.train_batch(x, mask, truth)


def test_recognizer_refusals_and_build():
    model = M.TransducerModel(params())
    for kw, err in (({'mode': 'beam'}, NotImplementedError), ({'lm': object()}, NotImplementedError),
                    ({'ngram_lm': object()}, NotImplementedError), ({'max_len': 0}, ValueError),
                    ({'max_symbols_per_frame': 0}, ValueError)):
        with pytest.raises(err):
            recognize.TransducerRecognizer(model, ngpu=0, **kw)
    args = argparse.Namespace(ngpu=0, max_len=50, mode='greedy', ngram_lm=None)
    rec = recognize.build_recognizer('transducer', model, None, args, None)
    assert isinstance(rec, recognize.TransducerRecognizer) and rec.max_len == 50 and rec.max_symbols_per_frame == 5
    with pytest.raises(NotImplementedError):
        recognize.build_recognizer('transducer', model, None, argparse.Namespace(ngpu=0, max_len=50, mode='beam'), None)


def test_model_restatement_loss_is_the_lattice_loss():
    """The whole-model restatement's loss equals torchaudio's rnnt_loss on the restatement's own joint logits."""
    p = params()
    torch.manual_seed(3)
    model = M.TransducerModel(p)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 60, 80, generator=g)
    mask = torch.arange(60)[None] < torch.tensor([60, 47])[:, None]
    truth = torch.tensor([[1, 5, 6, 9, 1], [1, 7, 1, 0, 0]])
    tlen = torch.tensor([4, 2])
    loss, _ = rnnt_ref.model_loss(x, mask, truth, tlen, sd, p)
    memory, lengths = rnnt_ref.encode_eval(x, mask, sd, p)
    tokens = torch.cat((torch.zeros(2, 1, dtype=torch.long), truth[:, 1:-1]), 1)
    logits = rnnt_ref.joint_logits(memory, rnnt_ref.predictor(tokens, sd, 1, 'bf16'), sd, 'bf16')
    want = TAF.rnnt_loss(logits, truth[:, 1:-1].int(), lengths.int(), (tlen - 1).int(), blank=0, reduction='mean')
    assert abs(float(loss) - float(want)) <= 1e-4 * abs(float(want))
