"""Encoder-forward time of the benchmark configuration (32 utterances x 1000 frames, cfg 2/3): median of 20 passes, CUDA events.
Used for A/B runs of two builds (OTB_LIB_PATH)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from opentransformer_b200.model import SpeechToText

dev = torch.device('cuda:0')
torch.manual_seed(0)
model = SpeechToText(bench.model_params()).eval().to(dev)
batches = [tuple(t.to(dev) for t in bench.synthetic_batch(32, i)) for i in range(8)]
with torch.no_grad():
    for i in range(4):
        model.encode_bf16(*batches[i % 8])
    torch.cuda.synchronize()
    ts = []
    for i in range(20):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        model.encode_bf16(*batches[i % 8])
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
ts.sort()
flop = 410e9
print(f'encoder forward median {ts[10]:.3f} ms, min {ts[0]:.3f} ms = '
      f'{flop / ts[10] / 1e9:.0f} TFLOP/s (410 GFLOP per 32 utterances)')
