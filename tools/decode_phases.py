"""Per-stage clock64 breakdown of one decode step of the persistent kernel (debug aid, GPU only).

The stamps come from the stamped instantiation, decode_group_kernel<true>, which otb_debug_decode_timing selects; the
production kernel (decode_group_kernel<false>) carries no stamp state.  Both run the same phases, but their registers are
allocated separately, so a phase's cycles here can differ slightly from the production kernel's."""
import sys, os, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from opentransformer_b200 import _lib
from opentransformer_b200.model import SpeechToText
from opentransformer_b200.recognize import BeamDecoder

dev = torch.device('cuda:0')
params = bench.model_params()
params['encoder']['n_blocks'] = 1
torch.manual_seed(0)
model = SpeechToText(params).eval().to(dev)
with torch.no_grad():
    model.decoder.output_layer.bias[1] = -1e4
x, mask = bench.synthetic_batch(32, 0)
x, mask = x.to(dev), mask.to(dev)
L = _lib.lib()
PH = ('qkv gemm', 'barrier', 'self-attn', 'W_o+LN1', 'q-proj', 'barrier', 'cross-attn', 'barrier', 'W_o2+LN2', 'barrier',
      'w1+glu', 'w2 partial', 'barrier', 'reduce+LN3', 'barrier')
NP = len(PH)
names = ['start', 'embed']
for l in range(6):
    names += [f'L{l} ' + n for n in PH]
names += ['logits', 'barrier', 'gather rows', 'row top-k', 'beam step', 'barrier']
with torch.no_grad():
    mem, lens, B, T2 = model.encode_bf16(x, mask)
    bd = BeamDecoder(model.decoder, B, 10, T2, 60, dev, use_graph=False, persistent=True)
    for step in [int(a) for a in (sys.argv[1:] or ['5', '50'])]:
        buf = torch.zeros(16 * 256, dtype=torch.int64, device=dev)
        for rep in range(2):
            bd.setup(mem, lens)
            L.otb_debug_decode_timing(ctypes.c_void_p(buf.data_ptr()) if rep == 1 else None, step)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); bd.run_persistent(60); e1.record()
            torch.cuda.synchronize()
        L.otb_debug_decode_timing(None, 0)
        allt = buf.cpu().view(16, 256)
        t = allt[0].tolist()
        n = len(names)
        print(f'=== step {step}: whole 60-step launch {e0.elapsed_time(e1):.2f} ms; step total {(t[n-1]-t[0])} cycles')
        agg = {}
        for i in range(1, n):
            dt = t[i] - t[i - 1]
            key = names[i].split(' ', 1)[1] if names[i].startswith('L') else names[i]
            agg[key] = agg.get(key, 0) + dt
        for k, v in agg.items():
            print(f'    {k:14s} {v:9d} cycles  {100.0 * v / (t[n-1]-t[0]):5.1f}%')
        print('    layer 0 detail:', [(names[i].split(' ', 1)[1], t[i] - t[i - 1]) for i in range(2, 2 + NP)])
        d = (allt[:, 1:n] - allt[:, :n - 1])                      # [cta, phase] durations of every CTA of group 0
        print('    layer 2, per phase (min / max over the 16 CTAs):',
              [(names[i].split(' ', 1)[1], int(d[:, i - 1].min()), int(d[:, i - 1].max())) for i in range(2 + 2 * NP, 2 + 3 * NP)])
        print('    tail, per phase (min / max over CTAs):', [(names[i], int(d[:, i - 1].min()), int(d[:, i - 1].max())) for i in range(n - 6, n)])
        sub = allt[:, 200:256]
        def dd(a, b):
            return [int(x) for x in (sub[:, b] - sub[:, a]).tolist()]
        print('    layer 2 W_o block, per CTA: rows in', dd(9, 10), 'GEMM', dd(10, 11))
        print('    beam step, per CTA: beam^2 top-k', dd(30, 31)[:12], 'ancestry', dd(31, 32)[:12], 'sync', dd(32, 33)[:12], 'state', dd(33, 35)[:12])
        print('    row top-k of hypothesis 0, per CTA: lane maxima', [int(x) for x in (sub[:, 52] - allt[:, n - 4]).tolist()][:12],
              'threshold', dd(52, 53)[:12], 'sum + candidates', dd(53, 54)[:12], 'ranking', dd(54, 55)[:12])
        print('    layer 2 self-attention, warp 0 task 1, per CTA: ancestry+q', dd(39, 40)[:6], 'issue 2 halves', dd(40, 41)[:6], 'wait half 0', dd(41, 42)[:6],
              'compute', dd(42, 43)[:6], 'wait half 1', dd(43, 44)[:6], 'compute', dd(44, 45)[:6], 'wait half 2', dd(45, 46)[:6], 'compute', dd(46, 47)[:6],
              'wait half 3', dd(47, 48)[:6], 'compute', dd(48, 49)[:6], 'merge+store', dd(50, 51)[:6])
        # inner stamps of the six group barriers of layer 2: stamp index of the barrier's entry = 2 + 2*NP + position of 'barrier' - 1
        bpos = [i for i, nme in enumerate(PH) if nme == 'barrier']
        rows = []
        for k, bp in enumerate(bpos):
            entry = allt[:, 2 + 2 * NP + bp - 1]      # stamp taken after the leading __syncthreads of gsync
            done = allt[:, 2 + 2 * NP + bp]
            a, b, c = allt[:, 212 + 3 * k], allt[:, 213 + 3 * k], allt[:, 214 + 3 * k]
            rows.append((PH[bp - 1], int((a - entry).median()), int((b - a).median()), int((c - b).median()), int((done - c).median())))
        print('    layer 2 group barriers (median over CTAs): after phase, fence+arrive (release), prefetch issue, wait (acquire), trailing sync:', rows)
