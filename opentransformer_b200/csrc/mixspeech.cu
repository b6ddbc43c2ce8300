// MixSpeech (otrans/train/trainer.py:155-201, DESIGN.md 4.5): the input of one MixSpeech micro-step.  With P = B / 2 pairs
// (an odd last utterance is dropped) and lambda ~ Beta(1/2, 1/2):
//   x_mix[p]    = lambda * x[2p] + (1 - lambda) * x[2p + 1]     over the whole padded [T, F], padded frames included
//   mask_mix[p] = mask[2p] | mask[2p + 1]
// lambda is drawn here, on the device, from (seed, step) (counter_rng.cuh), so a captured training step draws a fresh one
// on every replay and never sends it to the host.  The mix reproduces the reference's fp32 expression bit for bit: both
// products are rounded separately (1 - lambda rounded first) and then added, with no FMA contraction.  One thread writes
// lam_out = {lambda, lambda * scale, (1 - lambda) * scale}: the weight, and the loss-gradient scales of the two passes.
#include "counter_rng.cuh"
#include "launch.cuh"
#include "otb_internal.h"

namespace otb {

__device__ __forceinline__ float mix1(float a, float b, float lam, float om) { return __fadd_rn(__fmul_rn(a, lam), __fmul_rn(b, om)); }

__global__ void __launch_bounds__(256) mixspeech_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, int P, int T,
                                                        int F, const int* __restrict__ seed, const int* __restrict__ step, float scale,
                                                        float* __restrict__ lam_out, float* __restrict__ x_out,
                                                        uint8_t* __restrict__ mask_out, int vec4) {
    const float lam = mix_lambda((uint32_t)*seed, (uint32_t)*step);
    const float om = 1.0f - lam;
    const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)gridDim.x * blockDim.x;
    if (tid == 0) {
        lam_out[0] = lam;
        lam_out[1] = lam * scale;
        lam_out[2] = om * scale;
    }
    const size_t TF = (size_t)T * F;
    if (vec4) {
        const size_t row4 = TF / 4;
        const float4* x4 = reinterpret_cast<const float4*>(x);
        float4* o4 = reinterpret_cast<float4*>(x_out);
        for (size_t i = tid; i < (size_t)P * row4; i += nthr) {
            const size_t p = i / row4, j = i % row4;
            const float4 a = x4[2 * p * row4 + j], b = x4[(2 * p + 1) * row4 + j];
            o4[i] = make_float4(mix1(a.x, b.x, lam, om), mix1(a.y, b.y, lam, om), mix1(a.z, b.z, lam, om), mix1(a.w, b.w, lam, om));
        }
    } else {
        for (size_t i = tid; i < (size_t)P * TF; i += nthr) {
            const size_t p = i / TF, j = i % TF;
            x_out[i] = mix1(x[2 * p * TF + j], x[(2 * p + 1) * TF + j], lam, om);
        }
    }
    for (size_t i = tid; i < (size_t)P * T; i += nthr) {
        const size_t p = i / T, t = i % T;
        mask_out[i] = (uint8_t)((mask[2 * p * T + t] | mask[(2 * p + 1) * T + t]) != 0);
    }
}

const char* mixspeech_launch(cudaStream_t st, const float* x, const uint8_t* mask, int B, int T, int F, const int* seed, const int* step,
                             float scale, float* lam_out, float* x_out, uint8_t* mask_out) {
    if (B < 2 || T < 1 || F < 1) return "mixspeech: needs at least two utterances and a non-empty [T, F]";
    const int P = B / 2;
    const size_t TF = (size_t)T * F;
    const int vec4 = (TF % 4 == 0) && ((uintptr_t)x % 16 == 0) && ((uintptr_t)x_out % 16 == 0);
    const size_t work = (size_t)P * (vec4 ? TF / 4 : TF);
    size_t blocks = (work + 255) / 256;
    if (blocks > (size_t)(8 * num_sms())) blocks = 8 * num_sms();
    if (blocks < 1) blocks = 1;
    return launch<mixspeech_kernel>((unsigned)blocks, 256, 0, st, x, mask, P, T, F, seed, step, scale, lam_out, x_out, mask_out, vec4);
}

}  // namespace otb
