"""CUDA-graph capture and replay, host polls of device counters, and the LRU caches of per-geometry objects: the one place
the package touches torch.cuda.CUDAGraph (DESIGN.md 4.3).

The rule for every captured step: the first call runs eagerly and is real work (it also builds the lazy weight packs and
kernel attributes a capture must not create), then the same function is captured.  Capture records kernels without running
them, so no state has to be saved and restored around it, and no launch is counted for it.  A new weight pack (new device
pointers) makes the next call run eagerly and capture again."""
import inspect
import weakref

import torch
from torch.utils.weak import WeakIdKeyDictionary

from . import ops


def _weak(fn):
    """fn, holding a bound method's object weakly.  The object holds the CapturedStep that calls the method: a strong
    reference would make a cycle, which leaves a dropped search (its buffers and its graph's memory pool) to the cyclic
    garbage collector, and a collection that destroys a graph while another graph is being captured invalidates that
    capture."""
    if not inspect.ismethod(fn):
        return fn
    ref = weakref.WeakMethod(fn)
    return lambda *args: ref()(*args)


class CapturedStep:
    """A callable that returns what fn(*args) returns: fn eagerly on the first call (and the first after an object in
    keys() changed identity), captured right after it, and a replay of the capture on every later call, which must pass
    the same args (the graph reads the tensors of the capture).  use_graph=False runs fn eagerly every time.  graph is
    None until captured; launches is the kernel count of one replay, which every replay adds to ops.COUNTERS['launches']
    as an eager call of fn would.  keys() returns the weight packs whose device pointers the graph bakes in."""

    def __init__(self, fn, keys=lambda: (), use_graph=True):
        self.fn, self.keys, self.use_graph = _weak(fn), _weak(keys), use_graph
        self.graph = None
        self.launches = 0
        self._keys = self._out = None

    def __call__(self, *args):
        if not self.use_graph:
            return self.fn(*args)
        if self.graph is not None and all(a is b for a, b in zip(self._keys, self.keys())):
            self.graph.replay()
            ops.COUNTERS['launches'] += self.launches
            return self._out
        self.graph = None                   # frees the old graph (and its pool) before the new one is captured
        out = self.fn(*args)
        self._keys = tuple(self.keys())     # read after the eager call, which builds any pack that was out of date
        graph = torch.cuda.CUDAGraph()
        n0 = ops.COUNTERS['launches']
        with torch.cuda.graph(graph):
            self._out = self.fn(*args)
        self.launches = ops.COUNTERS['launches'] - n0
        ops.COUNTERS['launches'] = n0       # capture records, it does not launch
        self.graph = graph
        return out


_PINNED = WeakIdKeyDictionary()


def read_device(t):
    """A copy on the host of the small i32 device tensor t, after the work queued before it on the current stream.  The
    copy lands in pinned memory kept for t, and the thread SLEEPS on a blocking-sync event instead of spinning in
    cudaStreamSynchronize (`.item()`): a server keeps many search loops alive on few cores (16 lanes x 8 ranks on one
    host in bench.py).  The returned tensor is overwritten by the next read of t."""
    ent = _PINNED.get(t)
    if ent is None:
        ent = _PINNED[t] = (torch.empty(t.shape, dtype=t.dtype).pin_memory(), torch.cuda.Event(blocking=True))
    pin, ev = ent
    pin.copy_(t, non_blocking=True)
    ev.record()
    ev.synchronize()
    return pin


def lru_get(cache, key, limit, make):
    """cache[key], made by make() when missing, as the most recently used entry of the dict cache; before making one, the
    least recently used entries go until fewer than limit remain (None: no limit)."""
    val = cache.pop(key, None)
    if val is None:
        while limit is not None and len(cache) >= limit:
            cache.pop(next(iter(cache)))
        val = make()
    cache[key] = val
    return val
