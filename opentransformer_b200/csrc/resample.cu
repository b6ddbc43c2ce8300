// Band-limited resampling of a padded batch on the device, one rate pair per row: speed perturbation
// (otrans/data/audio.py:63-67,106-110, `resample_waveform(w, sr, int(sr * ratio))`, commented out there) and audio at
// another rate than the model's.  Row b equals torchaudio.functional.resample(x[b, :n_in[b]], orig[b], new[b]) with its
// defaults (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99), the filter Kaldi's resample_waveform used.
//
// With g = gcd(orig, new), o = orig / g, n = new / g, base = 0.99 min(o, n), output j = q n + p is
//     y[j] = sum_i x[i] h(t),   t = base (i n - j o) / (o n),   h(t) = cos^2(pi t / 12) sinc(pi t) base / o  for |t| < 6
// and h = 0 for |t| >= 6 (torchaudio clamps t to +-6, where the Hann window is cos^2(pi / 2) = 0).  Samples at i < 0 or
// i >= n_in[b] are zero, and the padding past n_in[b] is never read.  Only the taps with |t| < 6 are summed: phase p's
// start at k0(p) = floor(p o / n - W) + 1 relative to q o, W = 6 o / base, and there are at most ceil(2 W) of them.
// t comes from the integer numerator i n - j o (int64 relative to q o), never from i / o - j / n in float32: at 48 kHz
// x 60 s i / o is near 10^6 and float32 could not resolve the phase there.
//
// One CTA of 256 threads writes RS_CHUNK consecutive outputs of one row (grid: chunks x rows), thread tid the outputs
// tid, tid + 256, ...  When the row's phase table (n phases x T taps, T = ceil(2 W) + 1 rounded up to odd so that
// neighbouring phases fall in different banks) fits RS_TAB floats, the CTA first evaluates it into shared memory and
// then each output is T multiply-adds; otherwise each tap is evaluated where it is used.  Rows with orig == new are
// copied bit for bit.  The output length is ceil(n n_in / o) in integers; columns from there to `width` are zero.
#include <math.h>

#include "launch.cuh"
#include "otb_internal.h"

namespace otb {

static constexpr int RS_THREADS = 256;
static constexpr int RS_PER_THREAD = 16;
static constexpr int RS_CHUNK = RS_THREADS * RS_PER_THREAD;
static constexpr int RS_TAB = 8192;             // 32 KB: every phase of 44.1 / 22.05 kHz -> 16 kHz (5 600 / 6 080 floats)

struct RsRow {
    long long o, n;     // reduced rates
    int T;              // taps per output
    double W;           // half-width 6 o / base, in input samples
    double o_over_n;
    double tscale;      // base / (o n): t = numerator * tscale
    float hscale;       // base / o
};

__device__ __forceinline__ float rs_tap(long long num, const RsRow& r) {
    const float t = (float)((double)num * r.tscale);
    if (!(fabsf(t) < 6.f)) return 0.f;
    const float c = cospif(t * (1.f / 12.f));
    const float s = t == 0.f ? 1.f : sinpif(t) / (3.14159265358979f * t);
    return c * c * s * r.hscale;
}

// first tap of phase p, relative to q o
__device__ __forceinline__ long long rs_first(int p, const RsRow& r) { return (long long)floor((double)p * r.o_over_n - r.W) + 1; }

__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const float* __restrict__ x, int ldx, const int* __restrict__ n_in,
                                                              const int* __restrict__ orig, const int* __restrict__ new_rate,
                                                              float* __restrict__ y, int ldy, int* __restrict__ n_out, int width) {
    __shared__ float tab[RS_TAB];
    const int b = blockIdx.y, tid = threadIdx.x;
    const long long j0 = (long long)blockIdx.x * RS_CHUNK;
    const float* xr = x + (size_t)b * ldx;
    float* yr = y + (size_t)b * ldy;
    const int L = min(max(n_in[b], 0), ldx);
    const int r0 = orig[b], r1 = new_rate[b];
    long long out_len;
    RsRow r;
    if (r0 <= 0 || r1 <= 0) {
        out_len = 0;
    } else if (r0 == r1) {
        out_len = L;
    } else {
        int a = r0, c = r1;
        while (c != 0) { const int t = a % c; a = c; c = t; }
        r.o = r0 / a;
        r.n = r1 / a;
        const double base = 0.99 * (double)min(r.o, r.n);
        r.W = 6.0 * (double)r.o / base;
        r.T = ((int)ceil(2.0 * r.W) + 1) | 1;
        r.o_over_n = (double)r.o / (double)r.n;
        r.tscale = base / ((double)r.o * (double)r.n);
        r.hscale = (float)(base / (double)r.o);
        out_len = (r.n * L + r.o - 1) / r.o;
    }
    out_len = min(out_len, (long long)width);
    if (blockIdx.x == 0 && tid == 0) n_out[b] = (int)out_len;
    if (j0 >= width) return;
    if (j0 >= out_len || r0 <= 0 || r1 <= 0) {                 // the tail past the row's length
        for (long long j = j0 + tid; j < j0 + RS_CHUNK && j < width; j += RS_THREADS) yr[j] = 0.f;
        return;
    }
    if (r0 == r1) {                                             // torchaudio returns the waveform itself
        for (long long j = j0 + tid; j < j0 + RS_CHUNK && j < width; j += RS_THREADS) yr[j] = j < L ? xr[j] : 0.f;
        return;
    }
    const int n = (int)r.n, T = r.T;
    const bool table = (long long)n * T <= RS_TAB;
    if (table) {
        for (int e = tid; e < n * T; e += RS_THREADS) {
            const int p = e / T, k = e - p * T;
            tab[e] = rs_tap((rs_first(p, r) + k) * r.n - (long long)p * r.o, r);
        }
        __syncthreads();
    }
#pragma unroll 1
    for (int it = 0; it < RS_PER_THREAD; ++it) {
        const long long j = j0 + it * RS_THREADS + tid;
        if (j >= width) break;
        float v = 0.f;
        if (j < out_len) {
            const int p = (int)((unsigned)j % (unsigned)n);
            const long long q = (unsigned)j / (unsigned)n;
            const long long k0 = rs_first(p, r);
            const long long i0 = q * r.o + k0;
            if (table) {
                const float* h = tab + p * T;
                if (i0 >= 0 && i0 + T <= L) {
                    const float* xi = xr + i0;
#pragma unroll 4
                    for (int k = 0; k < T; ++k) v = fmaf(__ldg(xi + k), h[k], v);
                } else {
                    for (int k = 0; k < T; ++k) {
                        const long long i = i0 + k;
                        if (i >= 0 && i < L) v = fmaf(__ldg(xr + i), h[k], v);
                    }
                }
            } else {
                const long long num0 = k0 * r.n - (long long)p * r.o;
                for (int k = 0; k < T; ++k) {
                    const long long i = i0 + k;
                    if (i >= 0 && i < L) v = fmaf(__ldg(xr + i), rs_tap(num0 + k * r.n, r), v);
                }
            }
        }
        yr[j] = v;
    }
}

const char* resample_launch(cudaStream_t st, const float* x, int ldx, const int* n_in, const int* orig, const int* new_rate, float* y,
                            int ldy, int* n_out, int B, int width) {
    if (B < 1 || width < 1) return "resample: empty problem";
    if (B > 65535) return "resample: at most 65535 rows";
    if (ldx < 1 || ldy < width) return "resample: row pitch smaller than the row";
    const dim3 grid((unsigned)((width + (long long)RS_CHUNK - 1) / RS_CHUNK), B);
    return launch<resample_kernel>(grid, RS_THREADS, 0, st, x, ldx, n_in, orig, new_rate, y, ldy, n_out, width);
}

}  // namespace otb
