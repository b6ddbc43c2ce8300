"""CPU checks of opentransformer_b200/graphs.py: it is the only module that captures CUDA graphs, no search loop polls the
device with a spinning `.item()`, a CapturedStep does not keep the object whose methods it calls alive, and lru_get's
order and eviction."""
import gc
import os
import re
import weakref

from opentransformer_b200.graphs import CapturedStep, lru_get

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'opentransformer_b200')


def test_every_graph_is_captured_in_graphs_py():
    """Capture, replay and launch counting live in graphs.CapturedStep, so every captured step follows one rule; the
    searches poll the device through graphs.read_device, which sleeps on an event instead of spinning."""
    bad = []
    for name in sorted(os.listdir(PKG)):
        if not name.endswith('.py'):
            continue
        text = open(os.path.join(PKG, name)).read()
        if name != 'graphs.py':
            bad += [f'{name}: {w}' for w in ('CUDAGraph', 'cuda.graph(') if w in text]
        if name in ('recognize.py', 'ctc_fusion.py') and re.search(r'\.item\(\)', text):
            bad.append(f'{name}: .item()')
    assert not bad, 'outside graphs.py:\n' + '\n'.join(bad)


def test_lru_get_keeps_the_most_recent_entries():
    made = []

    def make(k):
        made.append(k)
        return k * 10

    cache = {}
    for k in (1, 2, 1, 3):
        assert lru_get(cache, k, 2, lambda: make(k)) == k * 10
    assert made == [1, 2, 3] and list(cache) == [1, 3]          # 1 was used after 2, so 2 went first
    unbounded = {}
    for k in range(5):
        lru_get(unbounded, k, None, lambda: make(k))
    assert list(unbounded) == list(range(5))


def test_captured_step_does_not_keep_its_owner_alive():
    """A search holds the CapturedStep of its own methods; a dropped search must go (with its graph and buffers) when its
    last reference does, not at a cyclic collection that could run during another capture."""
    class Search:
        def __init__(self):
            self.step = CapturedStep(self._work, self._packs, use_graph=False)

        def _work(self, x):
            return x + 1

        def _packs(self):
            return ()

    gc.disable()
    try:
        s = Search()
        assert s.step(1) == 2
        ref = weakref.ref(s)
        del s
        assert ref() is None
    finally:
        gc.enable()
