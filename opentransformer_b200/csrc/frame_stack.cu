// Low-frame-rate frame stacking (otrans/frontend/concat.py:11-56, DESIGN.md 4.14): the input of the concat front ends.
// Output row r = b * T2 + i of utterance b stacks the n input frames i*s .. i*s + n - 1, frame-major (column j*F + f, the
// nn.Unfold order); frames at or past T are zero, as the reference's zero padding makes them.  Because the n frames are
// consecutive rows of x, an output row is the contiguous slice x[b, i*s*F : i*s*F + n*F) -- a copy with a cast, not a
// gather.  Each thread writes 8 columns (one 16-byte store) from two 16-byte loads when F % 4 == 0 and x is 16-byte
// aligned.  The row is W = n*F rounded up to 8 wide (the GEMM's TMA row pitch); columns n*F .. W - 1 are zero.
// Optional epilogue y * alpha + table[i] (x*sqrt(d)+PE of an abs-pos encoder, module/pos.py:56) as two separately rounded
// fp32 operations, like the reference's expression.
#include "launch.cuh"
#include "otb_internal.h"

namespace otb {

__global__ void __launch_bounds__(256) frame_stack_kernel(const float* __restrict__ x, int T, int F, int n, int s, int T2, int W,
                                                          bf16* __restrict__ out, int ldo, float alpha,
                                                          const float* __restrict__ table, size_t rows, int vec4) {
    const int nF = n * F, groups = W / 8;
    const size_t total = rows * groups;
    for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (size_t)gridDim.x * blockDim.x) {
        const size_t r = g / groups;
        const int c0 = (int)(g % groups) * 8;
        const int b = (int)(r / T2), i = (int)(r % T2);
        const long long first = (long long)i * s;                                      // first stacked frame
        // columns [0, lim) come from x: inside the stack and before frame T
        const long long avail = first < T ? ((long long)T - first) * F : 0;
        const int lim = (int)(avail < nF ? avail : nF);
        const float* src = x + ((size_t)b * T + (size_t)(first < T ? first : 0)) * F;
        float v[8];
        if (vec4 && c0 + 8 <= lim) {
            const float4 a = *reinterpret_cast<const float4*>(src + c0), c = *reinterpret_cast<const float4*>(src + c0 + 4);
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = c.x; v[5] = c.y; v[6] = c.z; v[7] = c.w;
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = c0 + k < lim ? src[c0 + k] : 0.f;
        }
        if (table) {
            const float* tr = table + (size_t)i * nF;
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (c0 + k < nF) v[k] = __fadd_rn(__fmul_rn(v[k], alpha), tr[c0 + k]);
        } else if (alpha != 1.f) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = __fmul_rn(v[k], alpha);
        }
        __align__(16) bf16 o[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) o[k] = __float2bfloat16(v[k]);
        *reinterpret_cast<uint4*>(out + r * ldo + c0) = *reinterpret_cast<const uint4*>(o);
    }
}

const char* frame_stack_launch(cudaStream_t st, const float* x, int B, int T, int F, int n, int s, int T2, bf16* out, int ldo,
                               float alpha, const float* table) {
    if (B < 1 || T < 1 || F < 1 || n < 1 || s < 1 || T2 < 1) return "frame_stack: B, T, F, n, s and T2 must be >= 1";
    const long long nF = (long long)n * F;
    if (nF > (1 << 20)) return "frame_stack: n * F must be at most 2^20";
    const int W = (int)((nF + 7) / 8 * 8);
    if (ldo < W || ldo % 8) return "frame_stack: the output pitch must be a multiple of 8 and at least n * F rounded up to 8";
    if ((uintptr_t)out % 16) return "frame_stack: out must be 16-byte aligned";
    const int vec4 = (F % 4 == 0) && ((uintptr_t)x % 16 == 0);
    const size_t rows = (size_t)B * T2, work = rows * (W / 8);
    size_t blocks = (work + 255) / 256;
    if (blocks > (size_t)(8 * num_sms())) blocks = 8 * num_sms();
    return launch<frame_stack_kernel>((unsigned)blocks, 256, 0, st, x, T, F, n, s, T2, W, out, ldo, alpha, table, rows, vec4);
}

}  // namespace otb
