// Kernel launch with programmatic dependent launch (PDL).
//
// Small decode-step kernels spend a few microseconds inside their code but pay launch latency, CTA scheduling,
// shared-memory carve-out and the drain of the previous kernel serially, 52 times per beam step.  With the
// programmatic-stream-serialization attribute the next kernel of the stream is scheduled while its predecessor is still
// running: every kernel launched through launch_pdl() starts with PDL_TRIGGER() (dependents may be scheduled) and executes
// PDL_WAIT() (griddepcontrol.wait: the predecessor grid has completed and its memory is visible) before its first
// global-memory access, so correctness is unchanged while launch + prologue overlap the predecessor's tail.  Works inside
// CUDA-graph capture (programmatic dependency edges).
// Inside a captured CUDA graph the kernel-to-kernel edges already hide most of the launch latency, so the attribute is
// OFF by default (OTB_PDL=1 enables it); the two instructions are no-ops for a
// kernel launched without it.
#pragma once
#include <cuda_runtime.h>
#include <stdlib.h>

#include <utility>

namespace otb {

#define PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define PDL_WAIT() asm volatile("griddepcontrol.wait;" ::: "memory")

inline bool pdl_enabled() {
    static const bool on = [] {
        const char* e = getenv("OTB_PDL");
        return e && e[0] == '1';
    }();
    return on;
}

// One shared-memory carve-out for every hot-path kernel.  The L1 / shared-memory split of an SM is a per-kernel
// preference; kernels that prefer different splits cannot share an SM and switching the split needs the SM idle.  A decode
// step alternates 230 KB GEMMs, an 82 KB attention kernel, 34 KB / 17 KB / 0 KB SIMT kernels, and several utterance
// batches run such chains concurrently on separate streams -- so all of them ask for the maximum shared-memory carve-out
// (OTB_CARVEOUT=0 restores the driver default).
inline bool carveout_enabled() {
    static const bool on = [] {
        const char* e = getenv("OTB_CARVEOUT");
        return !(e && e[0] == '0');
    }();
    return on;
}

template <typename... KArgs>
inline void prefer_max_smem_carveout(void (*kern)(KArgs...)) {
    static thread_local const void* seen[64];
    static thread_local int nseen = 0;
    const void* key = reinterpret_cast<const void*>(kern);
    for (int i = 0; i < nseen; ++i)
        if (seen[i] == key) return;
    if (carveout_enabled() &&
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) != cudaSuccess)
        (void)cudaGetLastError();
    if (nseen < 64) seen[nseen++] = key;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    prefer_max_smem_carveout(kern);
    cudaLaunchConfig_t cfg;
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
    if (e != cudaSuccess) (void)cudaGetLastError();   // reported through the return value: do not leave it pending for a later launch
    return e;
}

}  // namespace otb
