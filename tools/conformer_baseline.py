"""Speed of the shipped conformer_baseline model (d_model 384, 4 heads of 96, 12 Conformer blocks, 6 decoder blocks) on one GPU:
  (a) encoder forward, 64 x 1000 frames (the geometry of bench.py's conformer_cfg4 extra), CUDA graph, CUDA events;
  (b) SpeechToTextRecognizer.recognize on the per-step CUDA-graph decode path, 32 x 1000 frames, beam 10, 60 steps (EOS bias
      -1e4 so every step runs): lone-batch latency (median wall time of one synchronised call) and utt/s over back-to-back calls;
  (c) the attention kernel alone at d_k 96 and d_k 64, B = 64, T' = 249, 4 heads, non-causal, full lengths: CUDA events over
      many launches, and the rate 4 T'^2 d_k flop per (batch, head).
Random init.  Prints the card name, power limit and max SM clock from the same run.

    python tools/conformer_baseline.py
"""
import copy
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from opentransformer_b200 import ops  # noqa: E402
from opentransformer_b200.model import SpeechToText  # noqa: E402
from opentransformer_b200.recognize import SpeechToTextRecognizer  # noqa: E402
from tests.test_head_dim_96 import CONFORMER_BASELINE  # noqa: E402

BF16_DENSE_PEAK = 989e12   # H100 SXM data sheet, dense BF16 (700 W card)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def build(dev):
    torch.manual_seed(1234)
    model = SpeechToText(copy.deepcopy(CONFORMER_BASELINE)).eval()
    with torch.no_grad():
        model.decoder.output_layer.bias[1] = -1e4          # no hypothesis ends: all 60 steps run
    return model.to(dev)


def encoder_forward(model, dev, B=64, passes=20):
    ring = [tuple(t.to(dev) for t in bench.synthetic_batch(B, i)) for i in range(4)]
    with torch.no_grad():
        sx, sm = ring[0][0].clone(), ring[0][1].clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                model.encode_bf16(sx, sm)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            model.encode_bf16(sx, sm)
        for _ in range(3):
            graph.replay()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(passes):
            sx.copy_(ring[i % 4][0])
            sm.copy_(ring[i % 4][1])
            graph.replay()
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / passes
    del graph
    return ms, B / (ms * 1e-3)


def recognize(model, dev, B=32, beam=10, max_len=60, calls=8):
    rec = SpeechToTextRecognizer(model, beam_width=beam, nbest=1, max_len=max_len, penalty=0.6, lamda=5, ngpu=1, persistent=False)
    batches = [tuple(t.to(dev) for t in bench.synthetic_batch(B, 100 + i)) for i in range(4)]
    for i in range(3):                                      # graph capture and first launches
        _, _, n = rec.recognize_ids(*batches[i % 4])
    assert n == max_len, n
    assert not next(iter(rec._decoders.values())).persistent
    lat = []
    for i in range(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rec.recognize_ids(*batches[i % 4])
        torch.cuda.synchronize()
        lat.append(time.perf_counter() - t0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(calls):
        rec.recognize_ids(*batches[i % 4])
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    return statistics.median(lat) * 1e3, B * calls / total


def attention_kernel(dev, d_k, B=64, T=249, H=4, launches=200):
    d = H * d_k
    qkv = (torch.randn(B * T, 3 * d, device=dev)).to(torch.bfloat16)
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    out = torch.empty(B * T, d, dtype=torch.bfloat16, device=dev)

    def run():
        ops.attention(qkv, qkv, qkv, B, H, T, T, kv_len=lens, q_col0=0, k_col0=d, v_col0=2 * d, out=out, d_k=d_k)
    for _ in range(10):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / launches * 1e3
    flop = 4.0 * T * T * d_k * B * H
    return us, flop / (us * 1e-6)


def main():
    if not torch.cuda.is_available():
        raise SystemExit('needs a GPU: nothing here is measured on the CPU')
    dev = torch.device('cuda:0')
    print(f'card: {card()}')
    model = build(dev)
    ms, ups = encoder_forward(model, dev)
    print(f'(a) encoder forward, 64 x 1000 frames: {ms:.2f} ms per batch = {ups:.0f} utt/s')
    lat, ups = recognize(model, dev)
    print(f'(b) recognize (graph path), 32 x 1000 frames, beam 10, 60 steps: lone-batch latency {lat:.1f} ms (median of 8), '
          f'{ups:.0f} utt/s over 8 back-to-back calls')
    for d_k in (96, 64):
        us, rate = attention_kernel(dev, d_k)
        print(f'(c) attn_tc_kernel d_k {d_k}, B 64, T\' 249, 4 heads, non-causal: {us:.1f} us per launch (mean of 200), '
              f'{rate / 1e12:.1f} TFLOP/s at 4 T\'^2 d_k flop per (b, h) = {100 * rate / BF16_DENSE_PEAK:.1f} % of the '
              f'989 TFLOP/s dense BF16 data-sheet peak')


if __name__ == '__main__':
    main()
