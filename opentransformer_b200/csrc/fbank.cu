// Log-mel filterbank features + utterance CMVN on the device: the step immediately in front of the hot path
// (otrans/data/audio.py:117-120 `ta.compliance.kaldi.fbank(wavform, num_mel_bins, sample_frequency, dither=0.0)` with Kaldi's
// defaults -- 25 ms frames / 10 ms shift, snip_edges, DC removal, pre-emphasis 0.97, povey window, power spectrum of the
// zero-padded power-of-two FFT, triangular mel filters on the Kaldi mel scale from 20 Hz to Nyquist, log(max(., eps)) -- and
// `normalization`, audio.py:22-24: (x - mean) / std over ALL elements of the utterance, unbiased std).
// torchaudio is a pip dependency of the reference (not vendored): the algorithm restated here is Kaldi's compute-fbank-feats
// as torchaudio.compliance.kaldi publishes it; parity is anchored on that function (tests/test_gpu_features.py).
//
// One CTA per frame, 256 threads; the frame (<= 2048 samples) lives in shared memory through DC removal,
// pre-emphasis, windowing and an in-place radix-2 FFT of n_fft = round_to_power_of_two(frame_len) points (Kaldi's
// padded_window_size); each thread runs the butterflies, bins and samples j = tid, tid + 256, ... of a stage, so at n_fft 512
// it runs exactly one butterfly per stage and one power bin.  The filterbank row of mel bin f covers fft bins [lo_f, hi_f).
// Volume perturbation (audio.py:112-114) scales the samples where they are loaded, before DC removal, as the reference scales
// the waveform before fbank; after the log the max(e, eps) floor would make it differ on silent frames.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"
#include "ptx.cuh"

namespace otb {

static constexpr int FB_MAX_NFFT = 2048;

__global__ void __launch_bounds__(256) fbank_kernel(const float* __restrict__ wave, int ld_wave, const int* __restrict__ n_samples,
                                                    const float* __restrict__ gain, const float* __restrict__ window,
                                                    const float* __restrict__ bank, const int* __restrict__ bank_range,
                                                    float* __restrict__ out, int Tmax, int F, int frame_len, int frame_shift,
                                                    int log2_nfft, float preemph, float eps) {
    __shared__ float sx[FB_MAX_NFFT];
    __shared__ float2 a[FB_MAX_NFFT];
    __shared__ float red[8];
    const int t = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int n = n_samples[b];
    const int n_frames = (n >= frame_len) ? 1 + (n - frame_len) / frame_shift : 0;     // snip_edges
    float* o = out + ((size_t)b * Tmax + t) * F;
    if (t >= n_frames) {       // padded frames are zeros (collate pads features with 0.0, data/loader.py:81)
        for (int f = tid; f < F; f += 256) o[f] = 0.f;
        return;
    }
    const int n_fft = 1 << log2_nfft, n_bins = n_fft / 2;
    const float g = gain != nullptr ? gain[b] : 1.f;
    const float* x = wave + (size_t)b * ld_wave + (size_t)t * frame_shift;
    // DC offset of the frame
    float s = 0.f;
    for (int i = tid; i < frame_len; i += 256) {
        const float v = x[i] * g;
        sx[i] = v;
        s += v;
    }
    s = warp_sum(s);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    float mean = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) mean += red[i];
    mean /= (float)frame_len;
    // pre-emphasis on the DC-free frame (first sample uses itself as predecessor), povey window, zero padding, bit reversal
    for (int i = tid; i < n_fft; i += 256) {
        float v = 0.f;
        if (i < frame_len) {
            const float cur = sx[i] - mean, prev = sx[i > 0 ? i - 1 : 0] - mean;
            v = (cur - preemph * prev) * window[i];
        }
        a[__brev((unsigned)i) >> (32 - log2_nfft)] = make_float2(v, 0.f);
    }
    __syncthreads();
#pragma unroll 1
    for (int st = 1; st <= log2_nfft; ++st) {
        const int half = 1 << (st - 1);
#pragma unroll 1
        for (int j = tid; j < n_bins; j += 256) {
            const int k = j & (half - 1);
            const int base = (j >> (st - 1)) << st;
            float sn, cs;
            sincospif(-(float)k / (float)half, &sn, &cs);
            const float2 u = a[base + k], v = a[base + k + half];
            const float2 w = make_float2(v.x * cs - v.y * sn, v.x * sn + v.y * cs);
            a[base + k] = make_float2(u.x + w.x, u.y + w.y);
            a[base + k + half] = make_float2(u.x - w.x, u.y - w.y);
        }
        __syncthreads();
    }
    // power spectrum of bins 0 .. n_fft/2 - 1 (the Nyquist bin is outside the filterbank), reusing sx
    for (int i = tid; i < n_bins; i += 256) sx[i] = a[i].x * a[i].x + a[i].y * a[i].y;
    __syncthreads();
    for (int f = tid; f < F; f += 256) {
        const int lo = bank_range[2 * f], hi = bank_range[2 * f + 1];
        const float* w = bank + (size_t)f * n_bins;
        float e = 0.f;
        for (int i = lo; i < hi; ++i) e = fmaf(w[i], sx[i], e);
        o[f] = logf(fmaxf(e, eps));
    }
}

// audio.py:22-24: std, mean = torch.std_mean(feature) over every element of the utterance (unbiased); (x - mean) / std.
// With gmean / gstd (per-bin vectors, audio.py:131-132 global CMVN) the statistics are given.  With noise [B, F]
// (`gaussian_noise`, audio.py:131-133: one vector per utterance, the same on every frame) noise[b] is added in the store of
// the normalised value; gmean 0 / gstd 1 make that store an exact copy, so the noise alone costs the same one pass.  One CTA
// per utterance; frames >= n_frames[b] stay zero.
__global__ void __launch_bounds__(512) utt_cmvn_kernel(float* __restrict__ x, int Tmax, int F, const int* __restrict__ n_frames,
                                                       const float* __restrict__ gmean, const float* __restrict__ gstd,
                                                       const float* __restrict__ noise) {
    __shared__ float red[16];
    __shared__ float bc;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = min(n_frames[b], Tmax) * F;
    float* p = x + (size_t)b * Tmax * F;
    const float* nz = noise != nullptr ? noise + (size_t)b * F : nullptr;
    if (gmean != nullptr) {
        for (int i = tid; i < n; i += 512) {
            float v = (p[i] - gmean[i % F]) / gstd[i % F];
            if (nz != nullptr) v += nz[i % F];
            p[i] = v;
        }
        return;
    }
    if (n < 2) return;
    float s = 0.f;
    for (int i = tid; i < n; i += 512) s += p[i];
    s = warp_sum(s);
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
        float t = 0.f;
        for (int i = 0; i < 16; ++i) t += red[i];
        bc = t / (float)n;
    }
    __syncthreads();
    const float mean = bc;
    float q = 0.f;
    for (int i = tid; i < n; i += 512) { const float d = p[i] - mean; q += d * d; }
    q = warp_sum(q);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = q;
    __syncthreads();
    if (tid == 0) {
        float t = 0.f;
        for (int i = 0; i < 16; ++i) t += red[i];
        bc = rsqrtf(t / (float)(n - 1));
    }
    __syncthreads();
    const float rstd = bc;
    for (int i = tid; i < n; i += 512) {
        float v = __fmul_rn(p[i] - mean, rstd);           // rounded before the noise is added, as normalization(x) + noise
        if (nz != nullptr) v += nz[i % F];
        p[i] = v;
    }
}

const char* fbank_launch(cudaStream_t st, const float* wave, int ld_wave, const int* n_samples, const float* gain, int B,
                         const float* window, const float* bank, const int* bank_range, float* out, int Tmax, int F, int frame_len,
                         int frame_shift, float preemph) {
    if (B < 1 || Tmax < 1 || F < 1) return "fbank: empty problem";
    if (frame_len < 2 || frame_len > FB_MAX_NFFT || frame_shift < 1)
        return "fbank: frame length must be 2 .. 2048 samples (a FFT of at most 2048 points: 25 ms at <= 81.9 kHz)";
    int log2_nfft = 1;                                    // Kaldi's round_to_power_of_two(frame_len)
    while ((1 << log2_nfft) < frame_len) ++log2_nfft;
    return launch<fbank_kernel>(dim3(Tmax, B), 256, 0, st, wave, ld_wave, n_samples, gain, window, bank, bank_range, out, Tmax, F,
                                frame_len, frame_shift, log2_nfft, preemph, 1.1920928955078125e-07f);
}
const char* utt_cmvn_launch(cudaStream_t st, float* x, int B, int Tmax, int F, const int* n_frames, const float* gmean, const float* gstd,
                            const float* noise) {
    if (B < 1 || Tmax < 1 || F < 1) return "cmvn: empty problem";
    if ((gmean == nullptr) != (gstd == nullptr)) return "cmvn: global mean / std must both be given";
    return launch<utt_cmvn_kernel>(B, 512, 0, st, x, Tmax, F, n_frames, gmean, gstd, noise);
}

}  // namespace otb
