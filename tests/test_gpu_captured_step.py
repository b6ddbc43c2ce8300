"""graphs.CapturedStep at every site that captures a CUDA graph: a graph run counts the kernel launches an eager run of
the same work counts (the eager first call included, the capture not); the training graph draws the dropout masks of the
eager trainer; and a transducer recognizer whose model weights change recaptures its search in place."""
import pytest
import torch

from opentransformer_b200 import ops, train
from opentransformer_b200.ctc_fusion import CTCFusedSearch
from opentransformer_b200.recognize import BeamDecoder, TransducerRecognizer

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def _launches(fn):
    """(kernel launches counted while fn runs, fn's return)."""
    n0 = ops.COUNTERS['launches']
    out = fn()
    return ops.COUNTERS['launches'] - n0, out


def test_beam_decoder_graph_counts_the_eager_launches():
    from tests.test_gpu_model import _batch, _build, _params
    model, _ = _build(_params(n_enc=1, n_dec=2))
    model.eval()
    x, mask = _batch(4, 240, 80, [240, 200, 111, 239])
    counts, outs = {}, {}
    with torch.no_grad():
        mem, lens, B, T2 = model.encode_bf16(x.to(DEV), mask.to(DEV))
        for use_graph in (False, True):
            bd = BeamDecoder(model.decoder, B, 5, T2, 10, DEV, use_graph=use_graph, keep_logp=False)
            counts[use_graph] = []
            for _ in range(2):                  # the first search spans the capture, the second replays every step
                bd.setup(mem, lens)
                counts[use_graph].append(_launches(lambda: bd.run(10))[0])
            outs[use_graph] = (bd.state.tok_hist.clone(), bd.state.scores.clone())
            assert (bd.step.graph is not None) == use_graph
    assert counts[True] == counts[False], counts
    assert all(torch.equal(a, b) for a, b in zip(outs[True], outs[False]))


@pytest.mark.parametrize('kind', ['transformer', 'rnn'])
def test_ctc_fused_search_graph_counts_the_eager_launches(kind):
    from tests.test_gpu_ctc_lm_fusion import B, K, T, _frames, _lm
    lm = _lm(kind, 5)
    lp, tok, in_len, _ = _frames(40)
    counts, outs = {}, {}
    for use_graph in (False, True):
        s = CTCFusedSearch(lm, B, 4, T, K, DEV, 0.5, 0.2, use_graph=use_graph)
        runs = [_launches(lambda: s.run(lp, tok, in_len)) for _ in range(2)]
        counts[use_graph], outs[use_graph] = [n for n, _ in runs], runs[-1][1]
        assert (s.frame.graph is not None) == use_graph
    assert counts[True] == counts[False], counts
    assert all(torch.equal(a, b) for a, b in zip(outs[True], outs[False]))


def _transducer_kw(mode, lm):
    kw = dict(mode=mode, max_len=30, lm=lm, lm_weight=0.5, beta=0.2)
    return dict(kw, beam_width=4, nbest=2) if mode == 'alsd' else kw


@pytest.mark.parametrize('lm_kind', [None, 'rnn'])
@pytest.mark.parametrize('mode', ['greedy', 'alsd'])
def test_transducer_search_graph_counts_the_eager_launches(mode, lm_kind):
    from tests.test_gpu_rnnt_lm_fusion import _lm, _setup
    model, x, mask = _setup()
    lm = None if lm_kind is None else _lm(lm_kind, 9)
    counts, outs = {}, {}
    with torch.no_grad():
        for use_graph in (False, True):
            rec = TransducerRecognizer(model, use_graph=use_graph, **_transducer_kw(mode, lm))
            runs = [_launches(lambda: [t.clone() for t in rec.recognize_ids(x, mask)]) for _ in range(2)]
            counts[use_graph], outs[use_graph] = [n for n, _ in runs], runs[-1][1]
            assert rec._search.steps > rec._search.STEPS, 'the search must replay its captured block'
            assert (rec._search.block.graph is not None) == use_graph
    assert counts[True] == counts[False], counts
    assert all(torch.equal(a, b) for a, b in zip(outs[True], outs[False]))


def _lm_trainer(use_graph, dropout=0.0, accum_steps=2):
    from tests.test_gpu_transformer_lm_train import _lm, _params
    lm, _ = _lm(_params(tied=True, dropout=dropout))
    tr = train.FusedTrainer(lm.train(), accum_steps=accum_steps, use_graph=use_graph)
    tr.drop_seed.fill_(12345)
    return tr


def test_fused_trainer_graph_counts_the_eager_launches():
    """Five micro-steps of one geometry: eager, eager and captured, then replays (two optimizer steps among them)."""
    from tests.test_gpu_transformer_lm_train import _batch
    batches = [_batch(4, 30, seed=s) for s in range(5)]
    _lm_trainer(False).step(batches[0][0].to(DEV), batches[0][1].to(DEV))   # the process's first step fills shared caches
    counts, losses = {}, {}
    for use_graph in (False, True):
        tr = _lm_trainer(use_graph)
        runs = [_launches(lambda: float(tr.step(x.to(DEV), y.to(DEV)))) for x, y in batches]
        counts[use_graph], losses[use_graph] = [n for n, _ in runs], [v for _, v in runs]
        assert len(tr._graphs) == use_graph
    assert counts[True] == counts[False], counts
    assert losses[True] == losses[False], losses


def test_fused_trainer_graph_draws_the_eager_dropout_masks():
    """With dropout, 4 micro-steps of one optimizer step (the weights do not move): the graph trainer's losses are the
    eager trainer's bit for bit, and both end on the same dropout seed."""
    from tests.test_gpu_transformer_lm_train import _batch
    batches = [_batch(4, 30, seed=s) for s in range(4)]
    losses, seeds = {}, {}
    for use_graph in (False, True):
        tr = _lm_trainer(use_graph, dropout=0.1, accum_steps=4)
        losses[use_graph] = [float(tr.step(x.to(DEV), y.to(DEV))) for x, y in batches]
        seeds[use_graph] = int(tr.drop_seed[0])
        assert len(tr._graphs) == use_graph
    print('losses with dropout: eager', losses[False], 'graph', losses[True])
    assert losses[True] == losses[False] and len(set(losses[True])) == 4
    assert seeds[True] == seeds[False]


@pytest.mark.parametrize('lm_kind', [None, 'transformer', 'rnn'])
@pytest.mark.parametrize('mode', ['greedy', 'alsd'])
def test_transducer_new_weights_recapture_in_place(mode, lm_kind):
    from tests.test_gpu_rnnt_lm_fusion import _lm, _setup
    from tests.test_gpu_transducer import _tie_free_model
    model, x, mask = _setup()
    lm = None if lm_kind is None else _lm(lm_kind, 9)
    rec = TransducerRecognizer(model, **_transducer_kw(mode, lm))
    with torch.no_grad():
        a = [t.clone() for t in rec.recognize_ids(x, mask)]
        s0, g0 = rec._search, rec._search.block.graph
        model.load_state_dict(_tie_free_model(12, x, mask).state_dict())
        b = [t.clone() for t in rec.recognize_ids(x, mask)]
        assert rec._search is s0 and g0 is not None and s0.block.graph is not None and s0.block.graph is not g0
        fresh = TransducerRecognizer(model, **_transducer_kw(mode, lm)).recognize_ids(x, mask)
    assert all(torch.equal(u, v) for u, v in zip(b, fresh))
    assert not all(torch.equal(u, v) for u, v in zip(a, b))
