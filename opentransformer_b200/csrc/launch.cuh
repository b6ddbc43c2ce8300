// The one way the library launches a kernel:  launch<kernel>(grid, block, dynamic smem, stream, args...)
//
// It returns nullptr or the CUDA error string, and clears the error it caused, so that a refused launch cannot be
// blamed on a later call.  Cluster > 1 launches thread-block clusters of that many CTAs along x; Cooperative launches a
// grid whose CTAs are all resident at once (the launch fails instead of queueing CTAs), for kernels with a grid barrier.
//
// Before the first launch of each kernel, prepare<kernel>() sets two of its function attributes, once per process (a
// function-local static of a template instantiated per kernel: C++ initialises it exactly once, even when several
// threads launch at the same time):
//   - the dynamic shared-memory cap: the largest the kernel can take, i.e. the device's opt-in per-block maximum less
//     the kernel's static shared memory.  A launch is then bounded by the hardware alone, whatever a later call asks
//     for (decode_self_attn sizes its shared memory by Lmax, logsoftmax_topk by V).
//   - the maximum shared-memory carve-out.  The L1 / shared-memory split of an SM is a per-kernel preference; kernels
//     that prefer different splits cannot share an SM, and switching the split needs the SM idle.  A decode step
//     alternates 230 KB GEMMs, an 82 KB attention kernel and 34 KB / 17 KB / 0 KB SIMT kernels, a training step puts
//     its element-wise kernels between GEMMs, and several utterance batches run such chains concurrently on separate
//     streams -- so every kernel asks for the same split.
#pragma once
#include <cuda_runtime.h>

#include <utility>

namespace otb {

template <auto Kern>
const char* prepare() {
    static const cudaError_t err = [] {
        int dev = 0, optin = 0;
        cudaFuncAttributes fa;
        cudaError_t e = cudaGetDevice(&dev);
        if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, Kern);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, optin - (int)fa.sharedSizeBytes);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(Kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) (void)cudaGetLastError();
        return e;
    }();
    return err == cudaSuccess ? nullptr : cudaGetErrorString(err);
}

template <auto Kern, unsigned Cluster = 1, bool Cooperative = false, typename... Args>
const char* launch(dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    static_assert(Cluster == 1 || !Cooperative, "a launch is either clustered or cooperative");
    if (const char* err = prepare<Kern>()) return err;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute cluster;
    if (Cluster > 1) {
        cluster.id = cudaLaunchAttributeClusterDimension;
        cluster.val.clusterDim.x = Cluster;
        cluster.val.clusterDim.y = 1;
        cluster.val.clusterDim.z = 1;
        cfg.attrs = &cluster;
        cfg.numAttrs = 1;
    }
    cudaLaunchAttribute coop;
    if (Cooperative) {
        coop.id = cudaLaunchAttributeCooperative;
        coop.val.cooperative = 1;
        cfg.attrs = &coop;
        cfg.numAttrs = 1;
    }
    const cudaError_t e = cudaLaunchKernelEx(&cfg, Kern, std::forward<Args>(args)...);
    if (e == cudaSuccess) return nullptr;
    (void)cudaGetLastError();
    return cudaGetErrorString(e);
}

}  // namespace otb
