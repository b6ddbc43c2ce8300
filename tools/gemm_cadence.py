"""k-block cadence of the GEMM mainloop in normal / MMA-only / TMA-only mode (debug aid, GPU only)."""
import sys, os, ctypes
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from opentransformer_b200 import ops, _lib
dev = torch.device('cuda:0')
L = _lib.lib()
buf = torch.zeros(256 * 8 + 256 * 2 * 64, dtype=torch.int64, device=dev)
for (M, N, K) in [(7968, 2048, 2048), (7968, 1024, 2048), (7968, 64, 2048)]:
    a = torch.randn(M, K, device=dev).to(torch.bfloat16)
    w = torch.randn(N, K, device=dev).to(torch.bfloat16)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    for mode in (0, 1, 2):
        L.otb_debug_gemm_mode(mode)
        for _ in range(2):
            ops.linear(a, w, None, ops.EPI_BIAS, out=out)
        torch.cuda.synchronize()
        buf.zero_()
        L.otb_debug_gemm_timing(ctypes.c_void_p(buf.data_ptr()))
        ops.linear(a, w, None, ops.EPI_BIAS, out=out)
        torch.cuda.synchronize()
        L.otb_debug_gemm_timing(None)
        kbt = buf[256 * 8:].view(256, 2, 64).cpu()
        ful = [int(v) for v in kbt[3, 1] if int(v) > 0]
        iss = [int(v) for v in kbt[3, 0] if int(v) > 0]
        d = [ful[i + 1] - ful[i] for i in range(8, min(len(ful) - 1, 30))]
        di = [iss[i + 1] - iss[i] for i in range(8, min(len(iss) - 1, 30))]
        print(f'M={M} N={N} K={K} mode={mode}: full-to-full cycles (kb 8..30): mean {sum(d)/max(len(d),1):.0f}  {d[:12]}   issue-to-issue mean {sum(di)/max(len(di),1):.0f}')
L.otb_debug_gemm_mode(0)
