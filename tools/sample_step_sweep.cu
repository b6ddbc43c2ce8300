// The CTA-width sweep of sample_step_kernel (DESIGN.md 4.11): one warp per row (32 threads) against 64, 128, 256 and 512
// threads per row, at the row counts a sampling decode launches (B x K = 32 x 4 at bench.py's training geometry, and
// 320) and V = 4234 (the shipped vocabulary) and 49152 (the largest taken).  Built and run by tools/sample_step_sweep.py.
//
// Each timed window is `steps` launches from step 0 with every row live (the <S/E> logit is -inf, so no row ends and every
// launch does the full pass), the state reset between windows outside the timing; CUDA events around each window, the
// median of `reps` windows per configuration, the configurations interleaved.  The drawn tokens of every width are
// compared with the 256-thread launch's: the arg-max does not depend on the reduction order, so they must be identical.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "../opentransformer_b200/csrc/beam.cu"

using namespace otb;

// the library's definition lives in gemm_tc.cu; the launcher that reads it is not used here (the sweep launches each width)
int otb::num_sms() {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
}

#define CK(x)                                                                                  \
    do {                                                                                       \
        cudaError_t e_ = (x);                                                                  \
        if (e_ != cudaSuccess) {                                                               \
            fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));        \
            exit(1);                                                                           \
        }                                                                                      \
    } while (0)

struct Bufs {
    BeamState st;
    float* logits;
    int* seed;
};

static Bufs make(int N, int V, int Lmax) {
    Bufs b;
    std::vector<float> h((size_t)N * V);
    unsigned x = 12345u;
    for (auto& v : h) {                           // a fixed pseudo-random logit table, |x| < 4
        x = x * 1664525u + 1013904223u;
        v = ((x >> 8) * (1.0f / 16777216.0f) - 0.5f) * 8.0f;
    }
    for (int n = 0; n < N; ++n) h[(size_t)n * V + EOS_ID] = -INFINITY;
    CK(cudaMalloc(&b.logits, h.size() * sizeof(float)));
    CK(cudaMemcpy(b.logits, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMalloc(&b.seed, sizeof(int)));
    CK(cudaMemset(b.seed, 0, sizeof(int)));
    b.st.N = N;
    b.st.beam = 1;
    b.st.Lmax = Lmax;
    CK(cudaMalloc(&b.st.tok_hist, (size_t)Lmax * N * sizeof(int)));
    CK(cudaMalloc(&b.st.par_hist, (size_t)Lmax * N * sizeof(int)));
    CK(cudaMalloc(&b.st.last_tok, (size_t)N * sizeof(long long)));
    CK(cudaMalloc(&b.st.scores, (size_t)N * sizeof(float)));
    CK(cudaMalloc(&b.st.flag, (size_t)N));
    CK(cudaMalloc(&b.st.anc, (size_t)2 * N * Lmax * sizeof(int)));
    CK(cudaMalloc(&b.st.ctrl, 4 * sizeof(int)));
    return b;
}

static void reset(const Bufs& b) {
    CK(cudaMemset(b.st.ctrl, 0, 4 * sizeof(int)));
    CK(cudaMemset(b.st.flag, 0, b.st.N));
    CK(cudaMemset(b.st.scores, 0, b.st.N * sizeof(float)));
    CK(cudaMemset(b.st.anc, 0, (size_t)2 * b.st.N * b.st.Lmax * sizeof(int)));
}

template <int T>
static float window(const Bufs& b, int V, int steps) {
    reset(b);
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    for (int s = 0; s < steps; ++s) {
        if (const char* err = launch<sample_step_kernel<T>>(dim3(b.st.N), dim3(T), 0, (cudaStream_t)0, b.logits, V, V, b.st,
                                                            (const int*)b.seed)) {
            fprintf(stderr, "launch: %s\n", err);
            exit(1);
        }
    }
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    CK(cudaEventDestroy(e0));
    CK(cudaEventDestroy(e1));
    return ms * 1000.f / steps;                   // microseconds per launch
}

static std::vector<int> tokens(const Bufs& b, int steps) {
    std::vector<int> h((size_t)steps * b.st.N);
    CK(cudaMemcpy(h.data(), b.st.tok_hist, h.size() * sizeof(int), cudaMemcpyDeviceToHost));
    return h;
}

int main(int argc, char** argv) {
    const int steps = 60, reps = argc > 1 ? atoi(argv[1]) : 21;
    const int Ns[] = {128, 320};
    const int Vs[] = {4234, 49152};
    printf("[");
    bool first = true;
    for (int N : Ns)
        for (int V : Vs) {
            Bufs b = make(N, V, steps);
            window<256>(b, V, steps);             // warm-up of every width
            window<32>(b, V, steps);
            window<64>(b, V, steps);
            window<128>(b, V, steps);
            window<512>(b, V, steps);
            window<256>(b, V, steps);
            const std::vector<int> ref = tokens(b, steps);
            std::vector<float> t[5];
            bool same[5] = {true, true, true, true, true};
            for (int r = 0; r < reps; ++r) {
                t[0].push_back(window<32>(b, V, steps));
                same[0] = same[0] && tokens(b, steps) == ref;
                t[1].push_back(window<64>(b, V, steps));
                same[1] = same[1] && tokens(b, steps) == ref;
                t[2].push_back(window<128>(b, V, steps));
                same[2] = same[2] && tokens(b, steps) == ref;
                t[3].push_back(window<256>(b, V, steps));
                same[3] = same[3] && tokens(b, steps) == ref;
                t[4].push_back(window<512>(b, V, steps));
                same[4] = same[4] && tokens(b, steps) == ref;
            }
            const int widths[5] = {32, 64, 128, 256, 512};
            for (int i = 0; i < 5; ++i) {
                std::sort(t[i].begin(), t[i].end());
                printf("%s{\"rows\": %d, \"V\": %d, \"threads_per_row\": %d, \"us_per_launch_median\": %.2f, \"min\": %.2f, "
                       "\"max\": %.2f, \"tokens_equal_to_256\": %s}",
                       first ? "" : ", ", N, V, widths[i], t[i][t[i].size() / 2], t[i].front(), t[i].back(),
                       same[i] ? "true" : "false");
                first = false;
            }
        }
    printf("]\n");
    return 0;
}
