// Common device/host helpers for libbv2 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cmath>
#include <string>
#include <stdexcept>
#include <cstdlib>

namespace bv2 {

// Activation layout used by every internal buffer ("c4"): [B][C/4][T][4] fp32 -- four consecutive
// channels of one time step form one 16-byte element; time is the next-fastest dimension.  Rationale
// (DESIGN.md): (1) a time-shifted window of a [C/4][T][4] tile is a pure 16-byte-granular address
// offset, so the k taps of a dilated Conv1d become k wgmma smem-descriptor start addresses over ONE
// staged tile (K-major, no-swizzle canonical layout with SBO=128 B); (2) accumulator-image epilogues (one thread per
// time row, channels in registers) store 16-byte vectors that are contiguous across a warp.
struct Act {
    float* p = nullptr;
    int B = 0, C = 0, T = 0;  // C multiple of 4
    __host__ __device__ size_t elems() const { return (size_t)B * C * T; }
};

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

#define BV2_CUDA(expr)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess)                                                                      \
            throw ::bv2::Error(-3, std::string(#expr) + ": " + cudaGetErrorString(_e));             \
    } while (0)

#define BV2_CHECK(cond, msg)                                                                        \
    do {                                                                                            \
        if (!(cond)) throw ::bv2::Error(-2, std::string("check failed: ") + #cond + " : " + (msg)); \
    } while (0)

__device__ __forceinline__ float tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
__device__ __forceinline__ float lrelu(float x, float slope) { return x > 0.f ? x : x * slope; }
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float softplusf_(float x) { return x > 20.f ? x : log1pf(expf(x)); }  // F.softplus threshold=20

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// Launch with programmatic stream serialization: the kernel may start while its predecessor in the stream drains; every
// kernel launched this way executes `griddepcontrol.wait` (pdl_wait()) before touching data produced upstream.
template <typename... KArgs, typename... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    BV2_CUDA(cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...));
}
// Same, with a thread-block cluster of cluster_x CTAs along x (grid.x must be a multiple of cluster_x)
template <typename... KArgs, typename... Args>
inline void launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_x, Args... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = (unsigned)cluster_x; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 2;
    BV2_CUDA(cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...));
}

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

}  // namespace bv2
