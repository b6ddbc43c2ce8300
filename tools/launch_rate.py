"""How many small dependent kernels per second can L concurrent CUDA-graph lanes push through one GPU?
Each lane = one stream replaying a graph of 52 tiny dependent kernels (the shape of one decode step)."""
import sys, os, threading, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from opentransformer_b200 import ops

dev = torch.device('cuda:0')
x = torch.randn(320, 256, device=dev).to(torch.bfloat16)


def make_lane():
    st = torch.cuda.Stream()
    a, b = x.clone(), torch.empty_like(x)
    with torch.cuda.stream(st):
        for _ in range(3):
            ops.scale_add_table(a, 1.0, out=b)
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            for i in range(26):
                ops.scale_add_table(a, 1.0, out=b)
                ops.scale_add_table(b, 1.0, out=a)
    return st, g


for L in (1, 2, 4, 8, 12):
    lanes = [make_lane() for _ in range(L)]
    torch.cuda.synchronize()
    reps = 200

    def worker(j):
        st, g = lanes[j]
        with torch.cuda.stream(st):
            for _ in range(reps):
                g.replay()
        st.synchronize()
    t0 = time.perf_counter()
    ts = [threading.Thread(target=worker, args=(j,)) for j in range(L)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    dt = time.perf_counter() - t0
    n = L * reps * 52
    print(f'lanes {L:2d}: {n} kernels in {dt*1e3:7.1f} ms -> {n/dt/1e3:8.1f} k kernels/s, {dt/n*1e6:5.2f} us per kernel aggregate, '
          f'{dt/(reps*52)*1e6:5.2f} us per kernel per lane')
