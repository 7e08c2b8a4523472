// Hopper tensor-core (wgmma) implicit-GEMM Conv1d on the c4 activation layout, fp32 accumulators in wgmma registers (one-tile kernel)
// or in a shared-memory image (persistent kernels).
// Replaces the 90 dilated MRF convolutions of the HiFi-GAN Generator (reference modules.py:296-309 via
// models.py:546-552) = 96 % of the MACs of SynthesizerTrn.infer, the ups (models.py:543-545) and the flow convs.
//
// GEMM view of one CTA tile:  D[128 time steps, N = Cout] += sum_{tap j} sum_{ci}  A_j[t, ci] * W_j[ci, co]
//   A_j[t, ci] = act(x[ci][t0 + t + j*dil - pad])  -- a time-shifted view of ONE staged activation tile.
// A staged operand chunk is [KC/G channel groups][R = 128*MT + (K-1)*dil rows][16 bytes], i.e. the K-major / no-swizzle
// wgmma canonical layout with SBO = 128 B (8 rows x 16 B) and LBO = R*16 B, so tap j is just the smem-descriptor start
// address advanced by j*dil*16 bytes: the im2col matrix is never materialised and each activation byte is fetched from
// HBM/L2 once per conv instead of K times.
//
// Operand types (template parameter F16):
//   F16 = 0  TF32 operands (kind::tf32, K = 8 per MMA, G = 4 fp32 channels per 16-byte group): the c4 activation tile is the
//            operand image; the prologue rounds it to TF32 in place (integer round-to-nearest: ALU pipe, not the XU pipe).
//   F16 = 1  FP16 operands (kind::f16, K = 16 per MMA, G = 8 channels per group), fp32 activations in HBM as before: the
//            prologue converts the staged fp32 c4 tile into a [KC/8][R][8 halves] image next to it.  FP16 has the same
//            11-bit significand as TF32 (identical rounding error), twice the tensor-pipe rate, half the shared-memory
//            operand bytes per MMA and half the L2->SM weight traffic.  Out-of-range values saturate (cvt.rn.satfinite) instead of becoming inf.
//
// Warp roles: warp 0 = TMA producer (cp.async.bulk, mbarrier complete_tx), one warpgroup (persistent kernels) or two (one-tile
// kernel, 64 rows each) at the end of the block = wgmma issuers, 4 warps = operand prologue (leaky-relu + operand conversion in smem, zero fill of the conv padding
// rows, fence.proxy.async), 4 warps (the same ones in the one-tile kernel) = epilogue (accumulator init with
// bias/residual, tail -> scale/mask -> coalesced 16-byte stores, one thread per row of the accumulator image), +1 weight-producer warp.
#pragma once
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>
#include <cuda_fp16.h>
#include "common.cuh"
#include "wgmma.cuh"

namespace bv2 {

struct TcConvW {
    float* w = nullptr;  // packed [Cout/nt N tiles][nchunks][K][KC/G][nt][G] (fp32 TF32-rounded, or halves): one contiguous smem image per stage
    int Cin = 0, Cout = 0, K = 0, KC = 0, nchunks = 0, nt = 0;
    int ups_u = 0, ups_cout = 0;  // polyphase ConvTranspose1d: Cout = ups_u * ups_cout columns (phase-major)
    int f16 = 0;                  // operand type of the packed image
};
struct TcEpi {
    float in_slope = 1.f;        // leaky-relu slope applied to the conv INPUT (1 = identity)
    int in_mask = 0;             // input rows t >= lens[b] read as zero
    int relu = 0;
    int res_mode = 0;            // 1: v += res ; 2: v = res - v
    const float* res = nullptr;  // residual, c4, res_C_total channels, first channel res_c_off
    int res_C_total = 0, res_c_off = 0;
    int accumulate = 0;          // v += y_old
    float out_scale = 1.f;
    int out_mask = 0;            // v *= (t < lens[b])
    const int* lens = nullptr;
    const float* bias_b = nullptr;  // per-batch bias row (speaker conditioning)
    int bias_b_stride = 0;
    int cin_off = 0, cout_off = 0;  // channel windows inside x / y (multiples of 4; of 8 for 16-bit tensors)
    int dil = 1;
    int t_begin = 0, t_end = -1;  // output window [t_begin, t_end) (t_end = -1: the whole output); a ConvTranspose window is a multiple of its stride
    int out_tf32 = 0;    // round the stored output to TF32 (RN): a TF32 consumer may then skip its operand prologue
    int skip_xform = 0;  // TF32: input already TF32-exact, no activation / mask / padding needed (K == 1)
    int in_f16 = 0;      // FP16: x is a 16-bit c8 tensor [B][C/8][T][8] (the operand image itself: no prologue; K == 1)
    int out_f16 = 0;     // store y as a 16-bit c8 tensor
    int gate = 0;        // WN gate fused into the tail (reference commons.py:98-105): columns (2c, 2c+1) hold the tanh / sigmoid pre-activations of
                         // channel c (weights interleaved at load time); y gets tanh(a) * sigmoid(b) as a 16-bit c8 tensor with Cout/2 channels
    const float* ln_gamma = nullptr; const float* ln_beta = nullptr;  // LayerNorm over the Cout channels of each time step fused into the
                                                                      // tail (one N tile = all channels; combine with res for norm(x + conv))
};

inline float tf32_rn_host(float x) {
    uint32_t u; std::memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) == 0x7f800000u) return x;
    u = (u + 0x1000u) & 0xffffe000u;  // round to nearest, ties away (== cvt.rna.tf32.f32)
    float r; std::memcpy(&r, &u, 4);
    return r;
}
inline uint16_t f16_rn_host(float x) {
    if (x > 65504.f) x = 65504.f;
    if (x < -65504.f) x = -65504.f;
    __half h = __float2half_rn(x);
    uint16_t u; std::memcpy(&u, &h, 2);
    return u;
}
inline float f16_round_host(float x) {
    uint16_t u = f16_rn_host(x); __half h; std::memcpy(&h, &u, 2);
    return __half2float(h);
}

// w: [Cout][Cin][K] fp32 (weight-norm already folded)
// nt = N tile (0: largest divisor of Cout that is a multiple of 16 and <= 128: a 128-column fp32 accumulator image is 66 KB of shared memory)
// kc = K chunk (channels per pipeline stage)
// fill = false: only the sizes / layout fields are computed and an all-zero image of the right size is handed to `up` (the engine's
// measuring pass and bv2_load_packed, where the image comes from a file)
inline TcConvW tc_pack_weights(std::function<float*(const std::vector<float>&)>& up, const std::vector<float>& w, int Cout, int Cin, int K, int nt = 0,
                               int f16 = 0, int kc = 0, bool fill = true) {
    TcConvW t; t.Cin = Cin; t.Cout = Cout; t.K = K; t.f16 = f16;
    if (!nt) { nt = std::min(Cout, 128); while (Cout % nt || nt % 16) nt -= 16; }
    if (!kc) kc = 32;
    t.KC = Cin >= kc ? kc : Cin;
    const int G = f16 ? 8 : 4;
    if (Cin % t.KC != 0 || t.KC % (2 * G) != 0 || Cout % 16 != 0 || Cout < 16)
        throw Error(-2, "tc_conv: unsupported channel counts " + std::to_string(Cin) + "->" + std::to_string(Cout));
    if (nt < 16 || nt > 256 || nt % 16 || Cout % nt) throw Error(-2, "tc_conv: bad N tile");
    t.nt = nt;
    t.nchunks = Cin / t.KC;
    const int ncg = t.KC / G;
    const size_t total = (size_t)Cin * K * Cout;
    std::vector<float> p(f16 ? (total + 1) / 2 : total);
    uint16_t* ph = reinterpret_cast<uint16_t*>(p.data());
    for (int tile = 0; fill && tile < Cout / nt; tile++)
        for (int c = 0; c < t.nchunks; c++)
            for (int j = 0; j < K; j++)
                for (int g = 0; g < ncg; g++)
                    for (int n = 0; n < nt; n++)
                        for (int e = 0; e < G; e++) {
                            const int ci = c * t.KC + g * G + e;
                            const float v = w[((size_t)(tile * nt + n) * Cin + ci) * K + j];
                            const size_t stage = ((size_t)tile * t.nchunks + c) * K + j;
                            const size_t idx = ((stage * ncg + g) * nt + n) * G + e;
                            if (f16) ph[idx] = f16_rn_host(v); else p[idx] = tf32_rn_host(v);
                        }
    t.w = up(p);
    return t;
}

// ConvTranspose1d(Cin->Cout, K, stride u, padding (K-u)/2) as a polyphase stride-1 conv (reference models.py:543-545):
//   out[t*u + r][co] = sum_m sum_ci x[t + floor((r+p)/u) - m][ci] * w[ci][co][(r+p)%u + m*u]
// -> an ordinary conv over input-rate time with Kp taps (union of the per-phase offsets), N = u*Cout columns ordered
// (r, co), structural zeros where a phase does not use a tap.  wT: [Cin][Cout][K] (weight-norm folded).
// Input rows t - half .. t + half feed the u outputs of input row t of the polyphase ConvTranspose1d (stride u, K taps, padding (K-u)/2).
inline int ups_half(int K, int u) {
    const int p = (K - u) / 2, taps = K / u;
    int omin = 1 << 30, omax = -(1 << 30);
    for (int r = 0; r < u; r++)
        for (int m = 0; m < taps; m++) { int o = (r + p) / u - m; omin = std::min(omin, o); omax = std::max(omax, o); }
    return std::max(-omin, omax);
}
inline TcConvW tc_pack_upsample(std::function<float*(const std::vector<float>&)>& up, const std::vector<float>& wT, int Cin, int Cout, int K, int u,
                                int kc = 0, int f16 = 0, bool fill = true, int nt_max = 128) {
    const int p = (K - u) / 2, taps = K / u;
    const int half = ups_half(K, u);
    const int Kp = 2 * half + 1;  // symmetric so that pad = (Kp-1)/2
    std::vector<float> w((size_t)u * Cout * Cin * Kp, 0.f);  // [N = u*Cout][Cin][Kp]
    for (int r = 0; fill && r < u; r++)
        for (int m = 0; m < taps; m++) {
            const int o = (r + p) / u - m, j = (r + p) % u + m * u, tap = o + half;
            for (int co = 0; co < Cout; co++)
                for (int ci = 0; ci < Cin; ci++)
                    w[(((size_t)(r * Cout + co)) * Cin + ci) * Kp + tap] = wT[((size_t)ci * Cout + co) * K + j];
        }
    int nt = std::min(u * Cout, nt_max);
    TcConvW t = tc_pack_weights(up, w, u * Cout, Cin, Kp, nt, f16, kc, fill);
    t.ups_u = u; t.ups_cout = Cout;
    return t;
}

struct TcParams {
    const float* x; float* y; const float* w; const float* bias; const float* res; const float* bias_b; const int* lens;
    int Cin_total, cin_off, Cout_total, cout_off, res_C_total, res_c_off, bias_b_stride;
    int nt;           // columns per N tile
    int T, B, K, dil, pad, KC, nchunks, R, nws, nas, MT;
    int t_begin, t_end;  // rows [t_begin, t_end) of the M axis (output time; input time of a ConvTranspose) are stored; t_end = 0: all T rows
    uint32_t a_stage_bytes, a_op_off, w_stage_bytes, acc_cols;  // acc_cols: columns of the accumulator image
    float in_slope, out_scale;
    int accumulate, relu, res_mode, in_mask, out_mask, ups_u, ups_cout;
    int out_tf32, skip_xform, in_f16, out_f16, gate;
    const float* ln_gamma; const float* ln_beta;
    uint32_t res_soff;          // LayerNorm tail only: byte offset (in dynamic shared memory) of the TMA-staged residual tile [nt/4][128 rows][16 B];
                                // 0 = residual pre-loaded into the accumulator by the epilogue warps (acc_init_tile)
    // batched-GEMM extensions (TF32 attention GEMMs of the fp32/tf32 engines): grid z = b * zsplit + h
    int zsplit;                 // 0/1: z == batch
    int x_batch_z, y_batch_z;   // 1: tensor's batch index is z (else b)
    int x_c_zstride, y_c_zstride;  // channel offset added per h
    long long w_zstride;        // packed-weight offset per z (floats)
    int w_mode;                 // 1: B operand rows come from a c4 activation tensor (K == 1): w = tensor base
    int w_ld, w_rows, w_c_total, w_c_off, w_c_zstride;
};

// Device-side error flags: a barrier timeout raises both and lets the kernel run to completion instead of trapping the context
// ("never abort across the ABI").  g_tc_err_dev lives in device memory (what waiting threads poll: an L2 hit, never PCIe --
// polling the host-mapped copy from every waiting thread slowed every kernel ~100x in the first round-2 run);
// g_tc_err_flag points to a pinned, host-mapped int the host reads without a CUDA call (set by tc_init_device()).
__device__ int g_tc_err_dev = 0;
__device__ int* g_tc_err_flag = nullptr;

namespace tc {
// Accumulators live in shared memory, in front of every tensor-core kernel's own buffers: an fp32 image [column][ACC_TS rows] of the
// 128-row tile, addressed like a tensor-memory column/lane pair (taddr = row << 16 | column; the kernels' accumulator base is 0).
// The persistent kernels' MMA warpgroup streams one 64-row x <= 64-column slice of it through registers per weight stage (wg_mma); the
// one-tile kernel's MMA warpgroups read it once before their first MMA and write it once after their last (tc_issuer); the epilogue threads
// own one row each and read / write whole runs of columns.  ACC_TS = 132: the stride keeps both access patterns free of bank
// conflicts (a warp's wgmma fragment touches rows r..r+7 of columns c, c+2, c+4, c+6: banks 8k + r).
constexpr uint32_t ACC_TS = 132;
__host__ __device__ constexpr uint32_t acc_img_bytes(uint32_t cols) { return (cols * ACC_TS * 4u + 1023u) & ~1023u; }
extern __shared__ __align__(1024) uint8_t bv2_dyn_smem[];
__device__ __forceinline__ float* acc_ptr(uint32_t taddr) {
    return reinterpret_cast<float*>(bv2_dyn_smem) + (size_t)(taddr & 0xffffu) * ACC_TS + (taddr >> 16);
}
// 32x32b-style accesses: lane i of the calling warp takes row (taddr >> 16) + i, columns (taddr & 0xffff) + 0 .. n-1
template <int N>
__device__ __forceinline__ void acc_st(uint32_t taddr, const uint32_t* v) {
    float* d = acc_ptr(taddr) + (threadIdx.x & 31);
#pragma unroll
    for (int i = 0; i < N; i++) d[i * ACC_TS] = __uint_as_float(v[i]);
}
template <int N>
__device__ __forceinline__ void acc_ld(uint32_t taddr, uint32_t* v) {
    const float* d = acc_ptr(taddr) + (threadIdx.x & 31);
#pragma unroll
    for (int i = 0; i < N; i++) v[i] = __float_as_uint(d[i * ACC_TS]);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
// Bounded wait: a protocol bug must never hang the GPU.  try_wait carries a suspend-time hint so a waiting thread sleeps in
// hardware instead of polling (with ~10 mostly-idle role warps per CTA, un-hinted polling consumed > 50 % of the SM issue
// slots).  On a timeout (~2 s) the device error flag is raised and the wait is abandoned: the kernel finishes with
// undefined data, the host sees the flag at its next read-back and reports BV2_ERR_INTERNAL; once the flag is up every
// later wait gives up after one poll round, so a broken launch drains in milliseconds.
__device__ __noinline__ bool mbar_wait_slow(uint32_t bar, uint32_t parity) {
    long long t0 = clock64();
    for (uint32_t it = 0;; it++) {
        uint32_t done;
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity), "r"(1000000u) : "memory");
        if (done) return true;
        if ((it & 0xf) == 0xf) {
            if (*reinterpret_cast<volatile int*>(&g_tc_err_dev)) return false;  // another wait already timed out: drain quickly
            if (clock64() - t0 > 4000000000ll) {
                *reinterpret_cast<volatile int*>(&g_tc_err_dev) = 1;
                int* f = g_tc_err_flag;
                if (f) *reinterpret_cast<volatile int*>(f) = 1;
                printf("bv2 tc_conv: mbarrier wait timeout (block %d,%d,%d thread %d bar %u parity %u)\n", blockIdx.x, blockIdx.y, blockIdx.z,
                       threadIdx.x, bar, parity);
                return false;
            }
        }
    }
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(bar), "r"(parity), "r"(1000000u) : "memory");
    if (!done) mbar_wait_slow(bar, parity);
}
// Bounded wait written as ONE asm block (no C++ control flow on a per-thread result, no call), used by every role of the wgmma
// kernels: a call anywhere in a kernel that issues wgmma makes ptxas serialise its wgmma pipeline (C7510), and a call inside the
// MMA loop also demotes the loop's descriptor state from uniform registers.  Same timeout protocol as mbar_wait_slow (error
// flags raised, wait abandoned), minus the printf.
__device__ __forceinline__ void mbar_wait_u(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t.reg .u32 n, e;\n\t.reg .u64 t0, t1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra DONE_%=;\n\t"
        "mov.u64 t0, %%clock64;\n\t"
        "mov.u32 n, 0;\n"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t"
        "@p bra DONE_%=;\n\t"
        "add.u32 n, n, 1;\n\t"
        "and.b32 e, n, 15;\n\t"
        "setp.ne.u32 p, e, 0;\n\t"
        "@p bra WAIT_%=;\n\t"
        "ld.volatile.global.u32 e, [%3];\n\t"
        "setp.ne.u32 p, e, 0;\n\t"
        "@p bra DONE_%=;\n\t"
        "mov.u64 t1, %%clock64;\n\t"
        "sub.u64 t1, t1, t0;\n\t"
        "setp.lt.u64 p, t1, 4000000000;\n\t"
        "@p bra WAIT_%=;\n\t"
        "st.volatile.global.u32 [%3], 1;\n\t"
        "ld.global.u64 t1, [%4];\n\t"
        "setp.ne.u64 p, t1, 0;\n\t"
        "@p st.volatile.global.u32 [t1], 1;\n"
        "DONE_%=:\n\t}"
        ::"r"(bar), "r"(parity), "r"(1000000u), "l"(&g_tc_err_dev), "l"(&g_tc_err_flag) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// K-major, no-swizzle shared-memory matrix descriptor (wgmma): start>>4 [0,14), LBO>>4 [16,30) = stride between core matrices along K,
// SBO>>4 [32,46) = stride between 8-row core-matrix groups along M / N, layout type 0 (no swizzle) [62,64)
__device__ __forceinline__ uint64_t make_desc(uint32_t addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((addr & 0x3ffffu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}
// One 64-row x NC-column slice of the accumulator: image -> registers (or zeros), nk MMAs, registers -> image.
template <int F16, int NC>
__device__ __forceinline__ void wg_slice(float* img, uint64_t ad, uint64_t bd, uint64_t a_kstep, uint64_t b_kstep, int nk, uint32_t acc) {
    float c[NC / 2];
    const int cq = 2 * (threadIdx.x & 3);
#pragma unroll
    for (int i = 0; i < NC / 8; i++) {
        const float* q = img + (size_t)(8 * i + cq) * ACC_TS;
        c[4 * i] = acc ? q[0] : 0.f; c[4 * i + 1] = acc ? q[ACC_TS] : 0.f; c[4 * i + 2] = acc ? q[8] : 0.f; c[4 * i + 3] = acc ? q[ACC_TS + 8] : 0.f;
    }
    wgmma_fence();
    for (int kk = 0; kk < nk; kk++) Wgmma<F16, NC>::mma(c, ad + (uint64_t)kk * a_kstep, bd + (uint64_t)kk * b_kstep);
    wgmma_commit();
    wgmma_wait0();
#pragma unroll
    for (int i = 0; i < NC / 8; i++) {
        float* q = img + (size_t)(8 * i + cq) * ACC_TS;
        q[0] = c[4 * i]; q[ACC_TS] = c[4 * i + 1]; q[8] = c[4 * i + 2]; q[ACC_TS + 8] = c[4 * i + 3];
    }
}
// D[128 rows x n columns at accumulator column d] (+)= sum_kk A(ad + kk*a_kstep) . B(bd + kk*b_kstep), run by all 128 threads of the
// MMA warpgroup.  M = 128 is two 64-row wgmma slices (A advanced by 8 SBO strides), N in slices of 64 / 32 / 16 columns (B advanced by
// n/8 SBO strides).  acc = 0: the accumulator starts from zero.
template <int F16>
__device__ __forceinline__ void wg_mma(uint32_t d, uint64_t ad, uint64_t bd, uint64_t a_kstep, uint64_t b_kstep, int nk, int n, uint32_t acc) {
    const int t = threadIdx.x & 127;
    const uint64_t a_sbo = (ad >> 32) & 0x3fffu, b_sbo = (bd >> 32) & 0x3fffu;
#pragma unroll 1
    for (int h = 0; h < 2; h++) {
        const uint64_t ah = ad + (uint64_t)(8 * h) * a_sbo;
        float* img = acc_ptr(d) + 64 * h + 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll 1
        for (int n0 = 0; n0 < n;) {
            const uint64_t bn = bd + (uint64_t)(n0 >> 3) * b_sbo;
            float* im = img + (size_t)n0 * ACC_TS;
            if (n - n0 >= 64) { wg_slice<F16, 64>(im, ah, bn, a_kstep, b_kstep, nk, acc); n0 += 64; }
            else if (n - n0 >= 32) { wg_slice<F16, 32>(im, ah, bn, a_kstep, b_kstep, nk, acc); n0 += 32; }
            else { wg_slice<F16, 16>(im, ah, bn, a_kstep, b_kstep, nk, acc); n0 += 16; }
        }
    }
}
// Signal an mbarrier once every MMA the warpgroup issued so far has completed and its accumulator slices are back in shared memory
// (named barrier 1 = the MMA warpgroup).
__device__ __forceinline__ void wg_commit(uint32_t bar) {
    asm volatile("bar.sync 1, 128;" ::: "memory");
    if ((threadIdx.x & 127) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// round-to-nearest (ties away) TF32 with two integer instructions: identical bits to cvt.rna.tf32.f32 for finite inputs,
// but issued on the ALU pipe instead of the XU pipe the cvt shares with the prologue's other conversions
__device__ __forceinline__ float to_tf32(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u); }
// two fp32 -> packed f16x2 (lo in bits [0,16)), round-to-nearest-even, saturating
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
    return r;
}

__device__ __forceinline__ int tc_t_end(const TcParams& p) { return p.t_end > 0 ? p.t_end : p.T; }

// Pre-load one 128-row x nt accumulator tile: bias (+ per-batch bias) (+/- residual) (+ previous output).
// All global loads of a 32-column batch are issued before the first image stores (memory-level parallelism: the
// epilogue warps are the only threads touching residual/output tensors).
// GEN = 1: generic epilogue (polyphase ConvTranspose scatter, per-batch bias, relu, 16-bit output); GEN = 0: plain conv
// epilogue.  The plain instantiation keeps the MRF convs (most of the launches) free of the generic tail's registers and branches.
template <int NG, int GEN>
__device__ __forceinline__ void acc_init_tile(const TcParams& p, uint32_t trow, int b, int t, int n0, int nt, int yb = -1, int coff = -1, bool skip_res = false) {
    const bool ok = t < tc_t_end(p);  // stores, residual reads and accumulate reads stay inside the window
    const size_t tstride = (size_t)p.T * ((GEN && p.ups_u) ? p.ups_u : 1);
    if (yb < 0) yb = b;
    if (coff < 0) coff = p.cout_off;
    const float4* resb = p.res ? reinterpret_cast<const float4*>(p.res) + (size_t)yb * (p.res_C_total / 4) * tstride : nullptr;
    const float4* ybp = reinterpret_cast<const float4*>(p.y) + (size_t)yb * (p.Cout_total / 4) * tstride;
    const float sg = p.res_mode == 1 ? 1.f : -1.f;  // mode 2: tail negates -> res - (conv + bias)
    for (int col0 = 0; col0 < nt; col0 += 4 * NG) {
        float4 o[NG];
        int cos[NG], tts[NG];
#pragma unroll
        for (int g = 0; g < NG; g++) {
            const int n = n0 + col0 + 4 * g;
            int co = n, tt = t;
            if (GEN && p.ups_u) { const int r = n / p.ups_cout; co = n - r * p.ups_cout; tt = t * p.ups_u + r; }
            cos[g] = co; tts[g] = tt;
            if (col0 + 4 * g < nt) {
                o[g] = p.bias ? *reinterpret_cast<const float4*>(p.bias + co) : make_float4(0.f, 0.f, 0.f, 0.f);
                if (GEN && p.bias_b) {
                    const float4 b2 = *reinterpret_cast<const float4*>(p.bias_b + (size_t)b * p.bias_b_stride + co);
                    o[g].x += b2.x; o[g].y += b2.y; o[g].z += b2.z; o[g].w += b2.w;
                }
            }
        }
        if (ok && p.res_mode && !(GEN && skip_res)) {
            float4 r[NG];
#pragma unroll
            for (int g = 0; g < NG; g++) if (col0 + 4 * g < nt) r[g] = resb[(size_t)((p.res_c_off + cos[g]) / 4) * tstride + tts[g]];
#pragma unroll
            for (int g = 0; g < NG; g++) if (col0 + 4 * g < nt) { o[g].x += sg * r[g].x; o[g].y += sg * r[g].y; o[g].z += sg * r[g].z; o[g].w += sg * r[g].w; }
        }
        if (ok && p.accumulate) {
            float4 a[NG];
#pragma unroll
            for (int g = 0; g < NG; g++) if (col0 + 4 * g < nt) a[g] = ybp[(size_t)((coff + cos[g]) / 4) * tstride + tts[g]];
#pragma unroll
            for (int g = 0; g < NG; g++) if (col0 + 4 * g < nt) { o[g].x += a[g].x; o[g].y += a[g].y; o[g].z += a[g].z; o[g].w += a[g].w; }
        }
#pragma unroll
        for (int h = 0; h < NG / 4; h++) {
            if (col0 + 16 * h < nt) {
                uint32_t v[16];
#pragma unroll
                for (int g = 0; g < 4; g++) {
                    v[4 * g] = __float_as_uint(o[4 * h + g].x); v[4 * g + 1] = __float_as_uint(o[4 * h + g].y);
                    v[4 * g + 2] = __float_as_uint(o[4 * h + g].z); v[4 * g + 3] = __float_as_uint(o[4 * h + g].w);
                }
                acc_st<16>(trow + (uint32_t)(col0 + 16 * h), v);
            }
        }
    }
}

// Drain one accumulator tile: the accumulator image -> [relu] -> scale/mask -> c4 global (16-byte stores, coalesced across a warp).
template <int NG, int GEN>
__device__ __forceinline__ void acc_tail_tile(const TcParams& p, uint32_t trow, int b, int t, int n0, int nt, int len, int yb = -1, int coff = -1) {
    const bool ok = t < tc_t_end(p);  // stores, residual reads and accumulate reads stay inside the window
    const size_t tstride = (size_t)p.T * ((GEN && p.ups_u) ? p.ups_u : 1);
    if (yb < 0) yb = b;
    if (coff < 0) coff = p.cout_off;
    float4* ybp = reinterpret_cast<float4*>(p.y) + (size_t)yb * (p.Cout_total / 4) * tstride;
    uint4* yhp = reinterpret_cast<uint4*>(p.y) + (size_t)yb * (p.Cout_total / 8) * tstride;  // 16-bit c8 view
    const float s = ((p.out_mask && t >= len) ? 0.f : p.out_scale) * (p.res_mode == 2 ? -1.f : 1.f);
    for (int col0 = 0; col0 < nt; col0 += 4 * NG) {
        uint32_t v[NG / 4][16];
#pragma unroll
        for (int h = 0; h < NG / 4; h++) if (col0 + 16 * h < nt) acc_ld<16>(trow + (uint32_t)(col0 + 16 * h), v[h]);
        if (!ok) continue;
#pragma unroll
        for (int h = 0; h < NG / 4; h++) {
            if (GEN && p.gate) {
                if (col0 + 16 * h < nt) {
                    float a[8];
#pragma unroll
                    for (int e = 0; e < 8; e++) {
                        const float ta = __uint_as_float(v[h][2 * e]), sb = __uint_as_float(v[h][2 * e + 1]);
                        a[e] = tanhf(ta) * (1.f / (1.f + expf(-sb))) * s;
                    }
                    uint4 o;
                    o.x = pack_h2(a[0], a[1]); o.y = pack_h2(a[2], a[3]); o.z = pack_h2(a[4], a[5]); o.w = pack_h2(a[6], a[7]);
                    yhp[(size_t)((coff + (n0 + col0 + 16 * h) / 2) / 8) * tstride + t] = o;
                }
                continue;
            }
            if (GEN && p.out_f16) {
                if (col0 + 16 * h < nt) {
                    float f[16];
#pragma unroll
                    for (int e = 0; e < 16; e++) { f[e] = __uint_as_float(v[h][e]); if (p.relu) f[e] = fmaxf(f[e], 0.f); f[e] *= s; }
#pragma unroll
                    for (int q = 0; q < 2; q++) {
                        const int co = n0 + col0 + 16 * h + 8 * q;
                        uint4 o;
                        o.x = pack_h2(f[8 * q], f[8 * q + 1]); o.y = pack_h2(f[8 * q + 2], f[8 * q + 3]);
                        o.z = pack_h2(f[8 * q + 4], f[8 * q + 5]); o.w = pack_h2(f[8 * q + 6], f[8 * q + 7]);
                        yhp[(size_t)((coff + co) / 8) * tstride + t] = o;
                    }
                }
                continue;
            }
#pragma unroll
            for (int g = 0; g < 4; g++) {
                if (col0 + 16 * h + 4 * g < nt) {
                    const int n = n0 + col0 + 16 * h + 4 * g;
                    int co = n, tt = t;
                    if (GEN && p.ups_u) { const int r = n / p.ups_cout; co = n - r * p.ups_cout; tt = t * p.ups_u + r; }
                    float4 o = make_float4(__uint_as_float(v[h][4 * g]), __uint_as_float(v[h][4 * g + 1]), __uint_as_float(v[h][4 * g + 2]),
                                           __uint_as_float(v[h][4 * g + 3]));
                    if (GEN && p.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                    o.x *= s; o.y *= s; o.z *= s; o.w *= s;
                    if (p.out_tf32) { o.x = to_tf32(o.x); o.y = to_tf32(o.y); o.z = to_tf32(o.z); o.w = to_tf32(o.w); }
                    ybp[(size_t)((coff + co) / 4) * tstride + tt] = o;
                }
            }
        }
    }
}

// Tail with a fused LayerNorm over the nt = Cout channels of each row (reference attentions.py:21-24 after the residual add of
// attentions.py:114,118): the accumulator already holds bias + residual + conv (accumulator-init fusion), so the row statistics
// are three passes over the shared-memory accumulator image instead of a separate kernel with an HBM round trip.
__device__ __forceinline__ void acc_tail_ln(const TcParams& p, uint32_t trow, int b, int t, int nt, int len, const float4* rs = nullptr) {
    // rs: this thread's row of the TMA-staged residual tile ([nt/4][128 rows] float4, already offset by the row); nullptr = the residual
    // was pre-loaded into the accumulator.  x = acc + residual is re-formed in each pass (shared-memory reads are cheap, the accumulator image is not written).
    const bool ok = t < tc_t_end(p);  // stores, residual reads and accumulate reads stay inside the window
    float4* ybp = reinterpret_cast<float4*>(p.y) + (size_t)b * (p.Cout_total / 4) * p.T;
    float s = 0.f;
    for (int c0 = 0; c0 < nt; c0 += 32) {
        uint32_t v[32];
        acc_ld<32>(trow + (uint32_t)c0, v);
        if (rs) {
#pragma unroll
            for (int g = 0; g < 8; g++) {
                const float4 r = rs[(size_t)(c0 / 4 + g) * 128];
                s += (__uint_as_float(v[4 * g]) + r.x) + (__uint_as_float(v[4 * g + 1]) + r.y) + (__uint_as_float(v[4 * g + 2]) + r.z) + (__uint_as_float(v[4 * g + 3]) + r.w);
            }
        } else {
#pragma unroll
            for (int e = 0; e < 32; e++) s += __uint_as_float(v[e]);
        }
    }
    const float mean = s / (float)nt;
    float q = 0.f;
    for (int c0 = 0; c0 < nt; c0 += 32) {
        uint32_t v[32];
        acc_ld<32>(trow + (uint32_t)c0, v);
        if (rs) {
#pragma unroll
            for (int g = 0; g < 8; g++) {
                const float4 r = rs[(size_t)(c0 / 4 + g) * 128];
                float d;
                d = __uint_as_float(v[4 * g]) + r.x - mean; q = fmaf(d, d, q);
                d = __uint_as_float(v[4 * g + 1]) + r.y - mean; q = fmaf(d, d, q);
                d = __uint_as_float(v[4 * g + 2]) + r.z - mean; q = fmaf(d, d, q);
                d = __uint_as_float(v[4 * g + 3]) + r.w - mean; q = fmaf(d, d, q);
            }
        } else {
#pragma unroll
            for (int e = 0; e < 32; e++) { const float d = __uint_as_float(v[e]) - mean; q = fmaf(d, d, q); }
        }
    }
    const float rstd = rsqrtf(q / (float)nt + 1e-5f);
    const float m = (p.out_mask && t >= len) ? 0.f : 1.f;
    for (int c0 = 0; c0 < nt; c0 += 16) {
        uint32_t v[16];
        acc_ld<16>(trow + (uint32_t)c0, v);
        if (!ok) continue;
#pragma unroll
        for (int g = 0; g < 4; g++) {
            const float4 ga = __ldg(reinterpret_cast<const float4*>(p.ln_gamma + c0 + 4 * g)), be = __ldg(reinterpret_cast<const float4*>(p.ln_beta + c0 + 4 * g));
            float4 x = make_float4(__uint_as_float(v[4 * g]), __uint_as_float(v[4 * g + 1]), __uint_as_float(v[4 * g + 2]), __uint_as_float(v[4 * g + 3]));
            if (rs) { const float4 r = rs[(size_t)(c0 / 4 + g) * 128]; x.x += r.x; x.y += r.y; x.z += r.z; x.w += r.w; }
            float4 o;
            o.x = ((x.x - mean) * rstd * ga.x + be.x) * m; o.y = ((x.y - mean) * rstd * ga.y + be.y) * m;
            o.z = ((x.z - mean) * rstd * ga.z + be.z) * m; o.w = ((x.w - mean) * rstd * ga.w + be.w) * m;
            ybp[(size_t)((p.cout_off + c0) / 4 + g) * p.T + t] = o;
        }
    }
}

// TF32 operand prologue of one staged activation chunk [ncg][R][4] (generic proxy), in place: leaky-relu + RN-TF32, zero
// rows outside [r_lo, r_hi).  The stage is contiguous, so the loop runs over flat 16-byte elements with 4 independent
// load->store chains per thread (the un-unrolled per-row loop exposed the full LDS latency on every element).
__device__ __forceinline__ void xform_stage(float4* A, int ncg, int R, int r_lo, int r_hi, float slope, int tid2) {
    const int total = ncg * R;
    int r[4];
#pragma unroll
    for (int u = 0; u < 4; u++) r[u] = (tid2 + 128 * u) % R;
    const int step = 512 % R;  // row advance per iteration (512 elements), R >= 128
    for (int i0 = tid2; i0 < total; i0 += 512) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = i0 + 128 * u;
            v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < total && r[u] >= r_lo && r[u] < r_hi) v[u] = A[i];
        }
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int i = i0 + 128 * u;
            if (i < total) {
                float4 o;
                o.x = to_tf32(lrelu(v[u].x, slope)); o.y = to_tf32(lrelu(v[u].y, slope));
                o.z = to_tf32(lrelu(v[u].z, slope)); o.w = to_tf32(lrelu(v[u].w, slope));
                A[i] = o;
            }
            r[u] += step;
            while (r[u] >= R) r[u] -= R;
        }
    }
}

// FP16 operand prologue: staged fp32 chunk S [2*ncg8][R][4] -> operand image O [ncg8][R][8 halves] (leaky-relu, RN-even
// saturating conversion, zero rows outside [r_lo, r_hi)).  Each thread owns rows tid2, tid2+128, ... and walks the channel
// groups four at a time (8 independent 16-byte shared loads in flight); consecutive lanes touch consecutive 16-byte
// elements on both sides: conflict free.
__device__ __forceinline__ void xform16_stage(const float4* S, uint4* O, int ncg8, int R, int r_lo, int r_hi, float slope, int tid2) {
    for (int r = tid2; r < R; r += 128) {
        const bool in = r >= r_lo && r < r_hi;
        for (int g0 = 0; g0 < ncg8; g0 += 4) {
            float4 v[4][2];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                v[u][0] = make_float4(0.f, 0.f, 0.f, 0.f); v[u][1] = v[u][0];
                if (in && g0 + u < ncg8) { v[u][0] = S[(size_t)(2 * (g0 + u)) * R + r]; v[u][1] = S[(size_t)(2 * (g0 + u) + 1) * R + r]; }
            }
#pragma unroll
            for (int u = 0; u < 4; u++) {
                if (g0 + u < ncg8) {
                    uint4 o;
                    o.x = pack_h2(lrelu(v[u][0].x, slope), lrelu(v[u][0].y, slope)); o.y = pack_h2(lrelu(v[u][0].z, slope), lrelu(v[u][0].w, slope));
                    o.z = pack_h2(lrelu(v[u][1].x, slope), lrelu(v[u][1].y, slope)); o.w = pack_h2(lrelu(v[u][1].z, slope), lrelu(v[u][1].w, slope));
                    O[(size_t)(g0 + u) * R + r] = o;
                }
            }
        }
    }
}

// Arrive on an mbarrier from thread 0 of the warpgroup if bar != 0 (bar = 0: nothing to release).  One asm block: a C++ branch here
// would make ptxas serialise the wgmma pipeline across it.
__device__ __forceinline__ void wg_release(uint32_t bar) {
    asm volatile("{\n\t.reg .pred p, e;\n\t.reg .u32 t;\n\tmov.u32 t, %%tid.x;\n\tand.b32 t, t, 127;\n\tsetp.eq.u32 e, t, 0;\n\t"
                 "setp.ne.and.u32 p, %0, 0, e;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(bar) : "memory");
}

// One k-step of a 64-row x NT-column fragment, issued as the 64 / 32 / 16-column slices wg_mma cuts the same N tile into (B advanced
// by the slice's first column: 8 columns per 128-byte SBO stride = one 16-byte unit per column).
template <int F16, int NT>
__device__ __forceinline__ void wg_mma_nt(float* d, uint64_t a, uint64_t b) {
    if constexpr (NT >= 64) { Wgmma<F16, 64>::mma(d, a, b); wg_mma_nt<F16, NT - 64>(d + 32, a, b + 64); }
    else if constexpr (NT >= 32) { Wgmma<F16, 32>::mma(d, a, b); wg_mma_nt<F16, NT - 32>(d + 16, a, b + 32); }
    else if constexpr (NT >= 16) Wgmma<F16, 16>::mma(d, a, b);
}
}  // namespace tc

// State the one-tile kernel's MMA issuer carries through its loops (all warpgroup-uniform except img, the thread's own fragment rows).
// Descriptors are kept as (constant high word, 32-bit low word), as in tc_gen.cuh.
struct TcIssue {
    uint32_t bar_ar, bar_ae, bar_wf, bar_we, bar_acc;     // first barrier of each group
    uint32_t a_lo_base, w_lo_base, a_stage16, w_stage16;  // descriptor low words of ring slot 0 (A: this warpgroup's 64 rows), slot strides
    uint32_t a_kstep, b_kstep, dil, nas, nws;
    int nchunks, K;
    uint64_t hi;
    float* img;  // accumulator image at (row of this thread's first fragment row, column 0)
};

// The issuer of one MMA warpgroup of k_tc_conv1d: 64 rows x NT columns of fp32 accumulators in registers (indexed by compile-time
// constants only), loaded once from the image the epilogue warps initialised (bias, residual, old output) and written back once for
// the tail.  Per output the fp32 sequence is the init value, then chunk c, tap j, k-step: the order of the image round trip it replaces.
// Each stage's MMAs are one wgmma group; once the previous group has completed (wait_group 1) its ring slots are released while the
// current one runs.
template <int F16, int NT, int NK>
__device__ __forceinline__ void tc_issuer(const TcIssue& q) {
    using namespace tc;
    float acc[NT / 2];
    const int cq = 2 * (threadIdx.x & 3);
#pragma unroll
    for (int i = 0; i < NT / 8; i++) {
        const float* s = q.img + (size_t)(8 * i + cq) * ACC_TS;
        acc[4 * i] = s[0]; acc[4 * i + 1] = s[ACC_TS]; acc[4 * i + 2] = s[8]; acc[4 * i + 3] = s[ACC_TS + 8];
    }
    uint32_t sa = 0, aph = 0, a_cur = q.a_lo_base;  // activation ring slot, parity, descriptor low word of the slot
    uint32_t sw = 0, wph = 0, w_cur = q.w_lo_base;  // weight ring
    uint32_t rel_w = 0, rel_a = 0;                  // slots the previous stage read: released once its MMAs have completed
    for (int c = 0; c < q.nchunks; c++) {
        mbar_wait_u(q.bar_ar + 8u * sa, aph);
        uint32_t a_tap = a_cur;
        for (int j = 0; j < q.K; j++, a_tap += q.dil) {
            mbar_wait_u(q.bar_wf + 8u * sw, wph);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < NK; kk++)
                wg_mma_nt<F16, NT>(acc, q.hi | (a_tap + (uint32_t)kk * q.a_kstep), q.hi | (w_cur + (uint32_t)kk * q.b_kstep));
            wgmma_commit();
            wgmma_wait1();
            wg_release(rel_w);
            wg_release(rel_a);
            rel_w = q.bar_we + 8u * sw;
            rel_a = j == q.K - 1 ? q.bar_ae + 8u * sa : 0u;
            w_cur += q.w_stage16;
            if (++sw == q.nws) { sw = 0; wph ^= 1u; w_cur = q.w_lo_base; }
        }
        a_cur += q.a_stage16;
        if (++sa == q.nas) { sa = 0; aph ^= 1u; a_cur = q.a_lo_base; }
    }
    wgmma_wait0();
    wg_release(rel_w);
    wg_release(rel_a);
#pragma unroll
    for (int i = 0; i < NT / 8; i++) {
        float* d = q.img + (size_t)(8 * i + cq) * ACC_TS;
        d[0] = acc[4 * i]; d[ACC_TS] = acc[4 * i + 1]; d[8] = acc[4 * i + 2]; d[ACC_TS + 8] = acc[4 * i + 3];
    }
    mbar_arrive(q.bar_acc);
}
// (N tile, k-steps per stage) dispatch as a tree of two-way branches (a switch would become a jump table: see tc_gen.cuh); the k-steps
// of a stage are a compile-time count because a runtime k-step loop makes ptxas insert warpgroup.arrive around its MMAs (C7519).
// tc_conv_plan admits these N tiles and K chunks.
template <int F16, int NK>
__device__ __forceinline__ void tc_issuer_nt(const TcIssue& q, int nt) {
    if (nt <= 48) {
        if (nt <= 16) tc_issuer<F16, 16, NK>(q);
        else if (nt <= 32) tc_issuer<F16, 32, NK>(q);
        else tc_issuer<F16, 48, NK>(q);
    } else if (nt <= 96) {
        if (nt <= 64) tc_issuer<F16, 64, NK>(q);
        else tc_issuer<F16, 96, NK>(q);
    } else {
        if (nt <= 128) tc_issuer<F16, 128, NK>(q);
        else tc_issuer<F16, 192, NK>(q);
    }
}
template <int F16>
__device__ __forceinline__ void tc_issuer_nk(const TcIssue& q, int nt, int nk) {
    if (nk <= 2) {
        if (nk == 1) tc_issuer_nt<F16, 1>(q, nt);
        else tc_issuer_nt<F16, 2>(q, nt);
    } else {
        if (F16 || nk == 4) tc_issuer_nt<F16, 4>(q, nt);
        else tc_issuer_nt<F16, 8>(q, nt);
    }
}
inline bool tc_one_tile_nt(int nt) { return nt == 16 || nt == 32 || nt == 48 || nt == 64 || nt == 96 || nt == 128 || nt == 192; }
// k-steps per weight stage (K chunk / 2 channel groups): 1, 2, 4 (FP16: K chunk <= 64) or 8 (TF32)
inline bool tc_one_tile_nk(int KC, int f16) { const int nk = KC / (f16 ? 16 : 8); return nk == 1 || nk == 2 || nk == 4 || (!f16 && nk == 8); }

// ------------------------------------------------------------------------------------------------------------
// One 128-row tile per CTA.  grid: (M blocks of 128 time steps, N tiles, B [* heads])
//
// Accumulator-init fusion: before the first MMA the epilogue warps pre-load  bias (+ per-batch bias) (+/- residual)
// (+ previous output when accumulating)  into the accumulator image while the first TMA loads are in
// flight; the two MMA warpgroups (64 rows each) load it into their registers, accumulate every stage there and write the result
// back once; the tail is only  the accumulator image -> [relu] -> scale/mask -> store.
// 512 threads: warp 0 activation producer, warps 2-5 operand prologue + accumulator init + tail, warp 6 weight producer, warps 8-15
// the two MMA warpgroups (warps 1 and 7 idle).
template <int GEN, int F16>
__global__ void __launch_bounds__(512, 1) k_tc_conv1d(TcParams p) {
    using namespace tc;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + acc_img_bytes(p.acc_cols);  // behind the accumulator image
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;  // shfl: warp-uniform for the compiler
    const int t0 = p.t_begin + blockIdx.x * 128, n0 = blockIdx.y * p.nt, z = blockIdx.z;
    const int zs = p.zsplit > 1 ? p.zsplit : 1;
    const int b = z / zs, hz = z - b * zs;
    const int xb = p.x_batch_z ? z : b, yb = p.y_batch_z ? z : b;
    const int cin_off = p.cin_off + hz * p.x_c_zstride, cout_off = p.cout_off + hz * p.y_c_zstride;
    const int nt = p.nt;
    uint8_t* sA = smem;
    const int NAS = p.nas;
    uint8_t* sW = smem + (size_t)NAS * p.a_stage_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sW + (size_t)p.nws * p.w_stage_bytes);
    // barrier map: a_full[NAS], a_ready[NAS], a_empty[NAS], w_full[nws], w_empty[nws], acc_full, acc_init, res_full
    const uint32_t bar0 = smem_u32(bars);
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
    const int B_AFULL = 0, B_AREADY = NAS, B_AEMPTY = 2 * NAS, B_WFULL = 3 * NAS, B_WEMPTY = 3 * NAS + p.nws, B_ACC = 3 * NAS + 2 * p.nws,
              B_INIT = B_ACC + 1, B_RES = B_ACC + 2;

    if (threadIdx.x == 0) {
        // a ring slot is free once both MMA warpgroups released it; the accumulators are back in the image once all 256 MMA threads stored theirs
        for (int i = 0; i < NAS; i++) { mbar_init(BAR(B_AFULL + i), 1); mbar_init(BAR(B_AREADY + i), 128); mbar_init(BAR(B_AEMPTY + i), 2); }
        for (int i = 0; i < p.nws; i++) { mbar_init(BAR(B_WFULL + i), 1); mbar_init(BAR(B_WEMPTY + i), 2); }
        mbar_init(BAR(B_ACC), 256);
        mbar_init(BAR(B_INIT), 128);
        mbar_init(BAR(B_RES), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t acc0 = 0;  // accumulator image base (acc_ptr)
    // Programmatic dependent launch: everything above (barrier init) overlapped the tail of the previous kernel in the stream.  Roles
    // that touch only static data do not wait for it: the weight producer fills its ring and, when the accumulator init is bias-only,
    // the epilogue warps pre-load the accumulators while the upstream kernel is still running.  Everybody else waits, then releases
    // the dependents (releasing them before the wait would let the whole rest of the stream become resident at once).
    // LayerNorm tail with a TMA-staged residual (p.res_soff): the residual tile is copied into shared memory by the activation producer
    // right after the PDL wait and added by the tail, so the accumulator init is bias-only (static data, runs ahead of the wait) and the
    // MMAs never wait for residual loads (pre-loading the residual into the accumulator means dependent rounds of float4 loads per
    // thread AFTER the wait, with the MMA warpgroup parked on the init barrier).
    const bool res_smem = GEN && p.res_soff != 0;
    const bool bias_only = (!p.res_mode || res_smem) && !p.accumulate;
    const bool static_role = (warp == 6 && !p.w_mode) || (warp >= 2 && warp <= 5 && bias_only);
    if (!static_role) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    }

    const int R = p.R;
    const int G = F16 ? 8 : 4;                                  // channels per 16-byte operand group
    const int ncg_in = (F16 && !p.in_f16) ? p.KC / 4 : p.KC / G;  // 16-byte groups per chunk in the GLOBAL tensor
    const int gdiv = (F16 && p.in_f16) ? 8 : 4;                 // channels per 16-byte group in the global tensor
    // rows r of the staged tile map to t = t0 - pad + r; rows outside [0, T) are the conv's zero padding
    const int r_lo = max(0, p.pad - t0);
    const int r_hi = min(R, p.T - (t0 - p.pad));

    if (warp == 0) {
        // ===== activation producer: lane 0 owns the mbarrier protocol, lanes 0..ncg_in-1 each issue one TMA bulk copy (one
        // contiguous run per channel group) so a chunk's copies are issued in parallel instead of serially by one thread
        const uint32_t row_bytes = (uint32_t)(r_hi - r_lo) * 16u;
        const uint4* xg = reinterpret_cast<const uint4*>(p.x);
        for (int c = 0; c < p.nchunks; c++) {
            const int sa = c % NAS;
            if (lane == 0) {
                mbar_wait_u(BAR(B_AEMPTY + sa), ((c / NAS) & 1) ^ 1);
                mbar_expect_tx(BAR(B_AFULL + sa), row_bytes * ncg_in);
            }
            __syncwarp();
            if (lane < ncg_in) {
                const uint4* src = xg + ((size_t)xb * (p.Cin_total / gdiv) + cin_off / gdiv + (size_t)c * ncg_in + lane) * p.T + (t0 - p.pad + r_lo);
                const uint32_t dst = smem_u32(sA + (size_t)sa * p.a_stage_bytes) + ((uint32_t)lane * R + (uint32_t)r_lo) * 16u;
                bulk_g2s(dst, src, row_bytes, BAR(B_AFULL + sa));
            }
            if (res_smem && c == min(NAS, p.nchunks) - 1) {
                // residual tile -> shared memory, one bulk copy per channel group (behind the first ring fill: the operand tiles gate the MMAs)
                const int nrows = min(128, p.T - t0);
                if (lane == 0) mbar_expect_tx(BAR(B_RES), (uint32_t)nrows * 16u * (uint32_t)(nt / 4));
                __syncwarp();
                const float4* rg = reinterpret_cast<const float4*>(p.res) + ((size_t)yb * (p.res_C_total / 4) + p.res_c_off / 4) * p.T + t0;
                for (int g = lane; g < nt / 4; g += 32)
                    bulk_g2s(smem_u32(smem + p.res_soff) + (uint32_t)g * 2048u, rg + (size_t)g * p.T, (uint32_t)nrows * 16u, BAR(B_RES));
            }
        }
    } else if (warp == 6) {
        if (p.w_mode) {
            // B operand = rows n0.. of a c4 activation tensor (attention keys): lanes issue one bulk copy per channel group
            const int ncg = p.KC / 4;
            const int nvalid = max(0, min(nt, p.w_rows - n0));
            const uint32_t rb = (uint32_t)nvalid * 16u;
            const float* wb = p.w + (((size_t)b * (p.w_c_total / 4) + (p.w_c_off + hz * p.w_c_zstride) / 4) * p.w_ld + n0) * 4;
            for (int c = 0; c < p.nchunks; c++) {
                const int sw = c % p.nws;
                if (lane == 0) {
                    mbar_wait_u(BAR(B_WEMPTY + sw), ((c / p.nws) & 1) ^ 1);
                    mbar_expect_tx(BAR(B_WFULL + sw), rb * ncg);
                }
                __syncwarp();
                if (nvalid && lane < ncg)
                    bulk_g2s(smem_u32(sW + (size_t)sw * p.w_stage_bytes) + (uint32_t)lane * nt * 16u, wb + (size_t)(c * ncg + lane) * p.w_ld * 4, rb,
                             BAR(B_WFULL + sw));
            }
        } else if (lane == 0) {
            // ===== weight producer: its own thread so the weight ring runs ahead across chunk boundaries
            // slot / parity / addresses carried incrementally (one stage per ~20 instructions: the producer has to out-run the MMA issuer)
            const uint8_t* src = reinterpret_cast<const uint8_t*>(p.w + (size_t)z * p.w_zstride + (size_t)blockIdx.y * p.nchunks * p.K * (p.w_stage_bytes / 4));
            const uint32_t bar_wf = BAR(B_WFULL), bar_we = BAR(B_WEMPTY), dst0 = smem_u32(sW), nws_u = (uint32_t)p.nws;
            uint32_t sw = 0, ph = 1u, dst = dst0;
            const int nst = p.nchunks * p.K;
            for (int i = 0; i < nst; i++, src += p.w_stage_bytes) {
                // (no griddepcontrol here: once the ring is full a slot only frees after MMAs ran, i.e. after the waiting roles saw the
                //  upstream kernel complete; the first launch_dependents of ANY thread releases the CTA's dependents, so this role stays silent)
                mbar_wait_u(bar_we + 8u * sw, ph);
                mbar_expect_tx(bar_wf + 8u * sw, p.w_stage_bytes);
                bulk_g2s(dst, src, p.w_stage_bytes, bar_wf + 8u * sw);
                dst += p.w_stage_bytes;
                if (++sw == nws_u) { sw = 0; ph ^= 1u; dst = dst0; }
            }
        }
    } else if (warp >= 8) {
        // ===== two MMA warpgroups (warps 8-11: rows 0-63, warps 12-15: rows 64-127 of the tile): all 128 threads of a warpgroup run
        // the issue loop together (wgmma is warpgroup-collective); per weight stage KC/(2G) k-steps of 64 rows x nt columns each
        const int wg = (warp - 8) >> 2;
        TcIssue q;
        q.bar_ar = BAR(B_AREADY); q.bar_ae = BAR(B_AEMPTY); q.bar_wf = BAR(B_WFULL); q.bar_we = BAR(B_WEMPTY); q.bar_acc = BAR(B_ACC);
        q.a_lo_base = (((smem_u32(sA) + p.a_op_off) & 0x3ffffu) >> 4) + 64u * (uint32_t)wg | (((uint32_t)R * 16u) >> 4) << 16;  // + 64 rows x 16 B
        q.w_lo_base = ((smem_u32(sW) & 0x3ffffu) >> 4) | (((uint32_t)nt * 16u) >> 4) << 16;
        q.a_stage16 = p.a_stage_bytes >> 4; q.w_stage16 = p.w_stage_bytes >> 4;
        q.a_kstep = 2u * (uint32_t)R; q.b_kstep = 2u * (uint32_t)nt;  // two channel groups per MMA
        q.dil = (uint32_t)p.dil; q.nas = (uint32_t)NAS; q.nws = (uint32_t)p.nws;
        q.nchunks = p.nchunks; q.K = p.K;
        q.hi = (uint64_t)(128u >> 4) << 32;  // SBO = 128 B
        q.img = acc_ptr(acc0) + 64 * wg + 16 * (warp & 3) + (lane >> 2);
        mbar_wait_u(BAR(B_INIT), 0);
        tc_issuer_nk<F16>(q, nt, p.KC / (2 * G));
    } else if (warp == 1 || warp == 7) {  // idle (the MMA warpgroups start at a warpgroup boundary)
    } else {
        const int tid2 = threadIdx.x - 64;
        const int q = warp & 3;
        // ===== accumulator init (overlaps the first TMA loads)
        acc_init_tile<4, GEN>(p, acc0 + ((uint32_t)(q * 32) << 16), b, t0 + q * 32 + lane, n0, nt, yb, cout_off, res_smem);
        mbar_arrive(BAR(B_INIT));
        if (bias_only) {  // the init above touched static data only; everything below reads / overwrites tensors of the upstream kernel
            asm volatile("griddepcontrol.wait;" ::: "memory");
            asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        }
        const int len = p.lens ? p.lens[b] : p.T;
        const int r_mask_hi = p.in_mask ? min(r_hi, len - (t0 - p.pad)) : r_hi;  // rows >= this read as zero (x * x_mask)
        // ===== operand prologue on the staged tile (generic proxy), then hand over to the async proxy
        const float slope = p.in_slope;
        for (int c = 0; c < p.nchunks; c++) {
            const int sa = c % NAS;
            mbar_wait_u(BAR(B_AFULL + sa), (c / NAS) & 1);
            uint8_t* st = sA + (size_t)sa * p.a_stage_bytes;
            if (F16) {
                if (!p.in_f16) xform16_stage(reinterpret_cast<const float4*>(st), reinterpret_cast<uint4*>(st + p.a_op_off), p.KC / 8, R, r_lo, r_mask_hi, slope, tid2);
                else if (r_lo > 0 || r_hi < R) {
                    // 16-bit operand image with taps: the conv's zero padding is not part of the tensor; clear those rows of the staged
                    // tile (the TMA copies covered rows [r_lo, r_hi) only); rows t >= len are zero in the tensor itself (producer's mask)
                    uint4* A = reinterpret_cast<uint4*>(st);
                    const int ncg = p.KC / 8, nz = r_lo + (R - r_hi);
                    for (int i = tid2; i < ncg * nz; i += 128) {
                        const int g = i / nz, k = i - g * nz;
                        A[(size_t)g * R + (k < r_lo ? k : r_hi + (k - r_lo))] = make_uint4(0u, 0u, 0u, 0u);
                    }
                }
            } else if (!p.skip_xform) {
                xform_stage(reinterpret_cast<float4*>(st), p.KC / 4, R, r_lo, r_mask_hi, slope, tid2);
            }
            fence_async_smem();
            mbar_arrive(BAR(B_AREADY + sa));
        }
        // ===== tail
        mbar_wait_u(BAR(B_ACC), 0);
        if (GEN && p.ln_gamma) {
            const float4* rs = nullptr;
            if (res_smem) { mbar_wait_u(BAR(B_RES), 0); rs = reinterpret_cast<const float4*>(smem + p.res_soff) + (q * 32 + lane); }
            acc_tail_ln(p, acc0 + ((uint32_t)(q * 32) << 16), b, t0 + q * 32 + lane, nt, len, rs);
        } else {
            acc_tail_tile<4, GEN>(p, acc0 + ((uint32_t)(q * 32) << 16), b, t0 + q * 32 + lane, n0, nt, len, yb, cout_off);
        }
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------------------
// Persistent variant for narrow layers (Cin <= 32: Generator stages 3/4 = 36 of the 90 MRF convs, the last ups).
// Those launches have thousands of 128-row tiles with only K * Cin/(2G) tiny MMAs each, so the one-tile-per-CTA kernel
// is bound by its per-tile latency chain (launch, accumulator setup, barrier init, TMA round trip, tail).  Here each CTA
//   * keeps ALL weight taps resident in shared memory (<= 45 KB, loaded once),
//   * walks tiles blockIdx.x, +gridDim.x, ... with a 3-deep TMA ring for the activation tiles (producer runs ahead),
//   * double-buffers the accumulator image: the epilogue warps pre-load tile i+1's accumulator (bias/residual) and
//     drain tile i-1 while the MMA warpgroup works on tile i.
// 512 threads: warp 0 producer, warps 2-5 operand prologue, warps 6-9 accumulator init + tail, warps 12-15 MMA warpgroup
// (warps 1, 10, 11 idle: the warpgroup starts at a warpgroup boundary).
template <int GEN, int F16>
__global__ void __launch_bounds__(512, 1) k_tc_conv1d_persist(TcParams p, int mtiles, int ntiles_total) {
    using namespace tc;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + acc_img_bytes(p.acc_cols);  // behind the accumulator image
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nt = p.nt, NAS = p.nas, R = p.R;
    const int G = F16 ? 8 : 4, ncg = p.KC / G, ncg_in = p.KC / 4;
    uint8_t* sWt = smem;                                   // resident weights: [K][ncg][nt][G]
    const uint32_t w_bytes = (uint32_t)(p.K * p.KC * nt * (F16 ? 2 : 4));
    uint8_t* sA = smem + ((w_bytes + 127u) & ~127u);
    uint64_t* bars = reinterpret_cast<uint64_t*>(sA + (size_t)NAS * p.a_stage_bytes);
    const uint32_t bar0 = smem_u32(bars);
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
    const int B_WFULL = 0, B_AFULL = 1, B_AREADY = 1 + NAS, B_AEMPTY = 1 + 2 * NAS, B_INIT = 1 + 3 * NAS, B_ACC = 3 + 3 * NAS;

    if (threadIdx.x == 0) {
        mbar_init(BAR(B_WFULL), 1);
        for (int i = 0; i < NAS; i++) { mbar_init(BAR(B_AFULL + i), 1); mbar_init(BAR(B_AREADY + i), 128); mbar_init(BAR(B_AEMPTY + i), 1); }
        for (int i = 0; i < 2; i++) { mbar_init(BAR(B_INIT + i), 128); mbar_init(BAR(B_ACC + i), 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t acc0 = 0;  // accumulator image base (acc_ptr)
    const int n_mine = (ntiles_total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;  // tiles of this CTA

    if (warp == 0) {
        if (lane == 0) {  // weights do not depend on the upstream kernel: load them before the PDL wait
            mbar_expect_tx(BAR(B_WFULL), w_bytes);
            bulk_g2s(smem_u32(sWt), p.w, w_bytes, BAR(B_WFULL));
        }
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        for (int i = 0; i < n_mine; i++) {
            const int tile = blockIdx.x + i * gridDim.x, b = tile / mtiles, t0 = p.t_begin + (tile - b * mtiles) * 128;
            const int r_lo = max(0, p.pad - t0), r_hi = min(R, p.T - (t0 - p.pad));
            const uint32_t row_bytes = (uint32_t)(r_hi - r_lo) * 16u;
            const int sa = i % NAS;
            if (lane == 0) {
                mbar_wait_u(BAR(B_AEMPTY + sa), ((i / NAS) & 1) ^ 1);
                mbar_expect_tx(BAR(B_AFULL + sa), row_bytes * ncg_in);
            }
            __syncwarp();
            if (lane < ncg_in) {
                const float* src = p.x + (((size_t)b * (p.Cin_total / 4) + p.cin_off / 4 + lane) * p.T + (t0 - p.pad + r_lo)) * 4;
                bulk_g2s(smem_u32(sA + (size_t)sa * p.a_stage_bytes) + ((uint32_t)lane * R + (uint32_t)r_lo) * 16u, src, row_bytes, BAR(B_AFULL + sa));
            }
        }
    } else if (warp >= 12) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        {  // the 128 threads of the MMA warpgroup run the issue loop together (wgmma is warpgroup-collective)
            const uint32_t a_lbo = (uint32_t)R * 16u, b_lbo = (uint32_t)nt * 16u;
            const uint64_t a_kstep = (uint64_t)(2u * (uint32_t)R), b_kstep = (uint64_t)(2u * (uint32_t)nt);
            const uint64_t b_tap = (uint64_t)((uint32_t)ncg * nt);  // next tap's weight tile, in 16-byte units
            const int nk = p.KC / (2 * G);
            const uint64_t b_desc0 = make_desc(smem_u32(sWt), b_lbo, 128u);
            mbar_wait_u(BAR(B_WFULL), 0);
            for (int i = 0; i < n_mine; i++) {
                const int sa = i % NAS, ab = i & 1;
                mbar_wait_u(BAR(B_INIT + ab), (i >> 1) & 1);
                mbar_wait_u(BAR(B_AREADY + sa), (i / NAS) & 1);
                const uint64_t a_desc0 = make_desc(smem_u32(sA + (size_t)sa * p.a_stage_bytes) + p.a_op_off, a_lbo, 128u);
                const uint32_t d = acc0 + (uint32_t)(ab * nt);
                uint64_t bd_tap = b_desc0;
                for (int j = 0; j < p.K; j++, bd_tap += b_tap) {
                    uint64_t ad = a_desc0 + (uint64_t)(uint32_t)(j * p.dil), bd = bd_tap;
                    wg_mma<F16>(d, ad, bd, a_kstep, b_kstep, nk, nt, 1u);
                }
                wg_commit(BAR(B_AEMPTY + sa));
                wg_commit(BAR(B_ACC + ab));
            }
        }
    } else if (warp == 1 || warp >= 10) {  // idle (the MMA warpgroup starts at a warpgroup boundary)
    } else if (warp < 6) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        // ===== operand prologue
        const int tid2 = threadIdx.x - 64;
        const float slope = p.in_slope;
        for (int i = 0; i < n_mine; i++) {
            const int tile = blockIdx.x + i * gridDim.x, b = tile / mtiles, t0 = p.t_begin + (tile - b * mtiles) * 128;
            const int len = p.lens ? p.lens[b] : p.T;
            const int r_lo = max(0, p.pad - t0), r_hi = min(R, p.T - (t0 - p.pad));
            const int r_mask_hi = p.in_mask ? min(r_hi, len - (t0 - p.pad)) : r_hi;
            const int sa = i % NAS;
            mbar_wait_u(BAR(B_AFULL + sa), (i / NAS) & 1);
            uint8_t* st = sA + (size_t)sa * p.a_stage_bytes;
            if (F16) xform16_stage(reinterpret_cast<const float4*>(st), reinterpret_cast<uint4*>(st + p.a_op_off), ncg, R, r_lo, r_mask_hi, slope, tid2);
            else xform_stage(reinterpret_cast<float4*>(st), ncg, R, r_lo, r_mask_hi, slope, tid2);
            fence_async_smem();
            mbar_arrive(BAR(B_AREADY + sa));
        }
    } else {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        // ===== accumulator init (tile i+1) and tail (tile i), double-buffered accumulator image
        const int q = warp & 3;
        auto init_tile = [&](int i) {
            const int tile = blockIdx.x + i * gridDim.x, b = tile / mtiles, t0 = p.t_begin + (tile - b * mtiles) * 128;
            acc_init_tile<4, GEN>(p, acc0 + ((uint32_t)(q * 32) << 16) + (uint32_t)((i & 1) * nt), b, t0 + q * 32 + lane, 0, nt);
            mbar_arrive(BAR(B_INIT + (i & 1)));
        };
        if (n_mine > 0) init_tile(0);
        for (int i = 0; i < n_mine; i++) {
            if (i + 1 < n_mine) init_tile(i + 1);
            const int tile = blockIdx.x + i * gridDim.x, b = tile / mtiles, t0 = p.t_begin + (tile - b * mtiles) * 128;
            const int len = p.lens ? p.lens[b] : p.T;
            mbar_wait_u(BAR(B_ACC + (i & 1)), (i >> 1) & 1);
            acc_tail_tile<4, GEN>(p, acc0 + ((uint32_t)(q * 32) << 16) + (uint32_t)((i & 1) * nt), b, t0 + q * 32 + lane, 0, nt, len);
        }
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------------------
// Persistent variant with STREAMED weights for wide layers (Cin >= 64).
// Each CTA walks tiles of MT*128 rows (n-tile fastest, so CTAs that share an activation tile run together and hit L2);
// the TMA producers run continuously over the flat (tile, chunk, tap) sequence, so the activation ring (NAS deep) and
// the weight ring (nws deep) stay full across tile boundaries; the accumulator image is double-buffered so the
// epilogue warps pre-load tile i+1's accumulator and drain tile i-1 while the MMA warpgroup is busy with tile i.
// The launcher uses MT = 1: two 128 x nt accumulator images already take up to 132 KB of shared memory.
// 512 threads: warp 0 activation producer, warps 2-5 operand prologue, warps 6-9 accumulator init + tail, warp 10 weight
// producer, warps 12-15 MMA warpgroup (warps 1 and 11 idle).
template <int GEN, int F16>
__global__ void __launch_bounds__(512, 1) k_tc_conv1d_pstream(TcParams p, int mtiles, int ntiles, int tiles_total) {
    using namespace tc;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + acc_img_bytes(p.acc_cols);  // behind the accumulator image
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nt = p.nt, NAS = p.nas, NWS = p.nws, R = p.R, NCH = p.nchunks, MT = p.MT;
    const int G = F16 ? 8 : 4, ncg = p.KC / G, ncg_in = p.KC / 4;
    uint8_t* sA = smem;
    uint8_t* sW = smem + (size_t)NAS * p.a_stage_bytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sW + (size_t)NWS * p.w_stage_bytes);
    const uint32_t bar0 = smem_u32(bars);
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
    const int B_AFULL = 0, B_AREADY = NAS, B_AEMPTY = 2 * NAS, B_WFULL = 3 * NAS, B_WEMPTY = 3 * NAS + NWS, B_INIT = 3 * NAS + 2 * NWS,
              B_ACC = B_INIT + 2;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NAS; i++) { mbar_init(BAR(B_AFULL + i), 1); mbar_init(BAR(B_AREADY + i), 128); mbar_init(BAR(B_AEMPTY + i), 1); }
        for (int i = 0; i < NWS; i++) { mbar_init(BAR(B_WFULL + i), 1); mbar_init(BAR(B_WEMPTY + i), 1); }
        for (int i = 0; i < 2; i++) { mbar_init(BAR(B_INIT + i), 128); mbar_init(BAR(B_ACC + i), 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t acc0 = 0;  // accumulator image base (acc_ptr)
    const int n_mine = (tiles_total - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    // tile -> (batch, m tile, n tile); n tile fastest
    auto decode = [&](int i, int& b, int& t0, int& ntile) {
        const int tile = blockIdx.x + i * gridDim.x;
        ntile = tile % ntiles;
        const int mm = tile / ntiles;
        b = mm / mtiles;
        t0 = p.t_begin + (mm - b * mtiles) * 128 * MT;
    };
    (void)ncg;

    if (warp == 0) {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        // ===== activation producer: runs up to NAS (tile, chunk) steps ahead of the MMA warp; copies issued by ncg_in lanes
        const int steps = n_mine * NCH;  // flat (tile, chunk) sequence
        for (int s_ = 0; s_ < steps; s_++) {
            int b, t0, ntile;
            decode(s_ / NCH, b, t0, ntile);
            const int c = s_ % NCH;
            const int r_lo = max(0, p.pad - t0), r_hi = min(R, p.T - (t0 - p.pad));
            const uint32_t row_bytes = (uint32_t)(r_hi - r_lo) * 16u;
            const int sa = s_ % NAS;
            if (lane == 0) {
                mbar_wait_u(BAR(B_AEMPTY + sa), ((s_ / NAS) & 1) ^ 1);
                mbar_expect_tx(BAR(B_AFULL + sa), row_bytes * ncg_in);
            }
            __syncwarp();
            if (lane < ncg_in) {
                const float* src = p.x + (((size_t)b * (p.Cin_total / 4) + p.cin_off / 4 + (size_t)c * ncg_in + lane) * p.T + (t0 - p.pad + r_lo)) * 4;
                bulk_g2s(smem_u32(sA + (size_t)sa * p.a_stage_bytes) + ((uint32_t)lane * R + (uint32_t)r_lo) * 16u, src, row_bytes, BAR(B_AFULL + sa));
            }
        }
    } else if (warp == 10) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        if (lane == 0) {
            // ===== weight producer: independent thread, so weight tiles stream up to NWS taps ahead across chunk and tile
            // boundaries (a single producer would serialise on the activation ring and bubble at every chunk).  Weights do
            // not depend on the upstream kernel: no PDL wait on this role.
            const int steps = n_mine * NCH;
            int wi = 0;
            const size_t wstage_f = p.w_stage_bytes / 4;
            const uint32_t bar_wf = BAR(B_WFULL), bar_we = BAR(B_WEMPTY), dst0 = smem_u32(sW), nws_u = (uint32_t)NWS;
            uint32_t sw = 0, ph = 1u, dst = dst0;
            for (int s_ = 0; s_ < steps; s_++) {
                int b, t0, ntile;
                decode(s_ / NCH, b, t0, ntile);
                const int c = s_ % NCH;
                const float* wsrc = p.w + ((size_t)ntile * NCH + c) * p.K * wstage_f;
                for (int j = 0; j < p.K; j++, wi++) {
                    mbar_wait_u(bar_we + 8u * sw, ph);
                    mbar_expect_tx(bar_wf + 8u * sw, p.w_stage_bytes);
                    bulk_g2s(dst, wsrc + (size_t)j * wstage_f, p.w_stage_bytes, bar_wf + 8u * sw);
                    dst += p.w_stage_bytes;
                    if (++sw == nws_u) { sw = 0; ph ^= 1u; dst = dst0; }
                }
            }
        }
    } else if (warp >= 12) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        {  // the 128 threads of the MMA warpgroup run the issue loop together (wgmma is warpgroup-collective)
            const uint32_t a_lbo = (uint32_t)R * 16u, b_lbo = (uint32_t)nt * 16u;
            const uint64_t a_kstep = (uint64_t)(2u * (uint32_t)R), b_kstep = (uint64_t)(2u * (uint32_t)nt);
            const int nk = p.KC / (2 * G);
            const uint64_t a_stage16 = (uint64_t)(p.a_stage_bytes >> 4), w_stage16 = (uint64_t)(p.w_stage_bytes >> 4);
            const uint64_t a_desc_base = make_desc(smem_u32(sA) + p.a_op_off, a_lbo, 128u), b_desc_base = make_desc(smem_u32(sW), b_lbo, 128u);
            const uint32_t bar_ar = BAR(B_AREADY), bar_ae = BAR(B_AEMPTY), bar_wf = BAR(B_WFULL), bar_we = BAR(B_WEMPTY);
            const uint32_t nas_u = (uint32_t)NAS, nws_u = (uint32_t)NWS;
            uint32_t sa = 0, aph = 0, sw = 0, wph = 0;
            uint64_t a_cur = a_desc_base, b_cur = b_desc_base;
            for (int i = 0; i < n_mine; i++) {
                const int ab = i & 1;
                mbar_wait_u(BAR(B_INIT + ab), (i >> 1) & 1);
                const uint32_t d0 = acc0 + (uint32_t)(ab * MT * nt);
                for (int c = 0; c < NCH; c++) {
                    mbar_wait_u(bar_ar + 8u * sa, aph);
                    uint64_t a_tap = a_cur;
                    for (int j = 0; j < p.K; j++, a_tap += (uint64_t)(uint32_t)p.dil) {
                        mbar_wait_u(bar_wf + 8u * sw, wph);
                        for (int mt = 0; mt < MT; mt++)
                            wg_mma<F16>(d0 + (uint32_t)(mt * nt), a_tap + (uint64_t)(uint32_t)(mt * 128), b_cur, a_kstep, b_kstep, nk, nt, 1u);
                        wg_commit(bar_we + 8u * sw);
                        b_cur += w_stage16;
                        if (++sw == nws_u) { sw = 0; wph ^= 1u; b_cur = b_desc_base; }
                    }
                    wg_commit(bar_ae + 8u * sa);
                    a_cur += a_stage16;
                    if (++sa == nas_u) { sa = 0; aph ^= 1u; a_cur = a_desc_base; }
                }
                wg_commit(BAR(B_ACC + ab));
            }
        }
    } else if (warp == 1 || warp == 11) {  // idle (the MMA warpgroup starts at a warpgroup boundary)
    } else if (warp < 6) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        // ===== operand prologue over the flat (tile, chunk) sequence
        const int tid2 = threadIdx.x - 64;
        const float slope = p.in_slope;
        const int steps = n_mine * NCH;
        for (int s_ = 0; s_ < steps; s_++) {
            int b, t0, ntile;
            decode(s_ / NCH, b, t0, ntile);
            const int len = p.lens ? p.lens[b] : p.T;
            const int r_lo = max(0, p.pad - t0), r_hi = min(R, p.T - (t0 - p.pad));
            const int r_mask_hi = p.in_mask ? min(r_hi, len - (t0 - p.pad)) : r_hi;
            const int sa = s_ % NAS;
            mbar_wait_u(BAR(B_AFULL + sa), (s_ / NAS) & 1);
            uint8_t* st = sA + (size_t)sa * p.a_stage_bytes;
            if (F16) xform16_stage(reinterpret_cast<const float4*>(st), reinterpret_cast<uint4*>(st + p.a_op_off), p.KC / 8, R, r_lo, r_mask_hi, slope, tid2);
            else xform_stage(reinterpret_cast<float4*>(st), p.KC / 4, R, r_lo, r_mask_hi, slope, tid2);
            fence_async_smem();
            mbar_arrive(BAR(B_AREADY + sa));
        }
    } else {
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        // ===== accumulator init (tile i+1) and tail (tile i), double-buffered accumulator image
        const int q = warp & 3;
        auto init_tile = [&](int i) {
            int b, t0, ntile;
            decode(i, b, t0, ntile);
            const int n0 = ntile * nt;
            for (int mt = 0; mt < MT; mt++)
                acc_init_tile<8, GEN>(p, acc0 + ((uint32_t)(q * 32) << 16) + (uint32_t)(((i & 1) * MT + mt) * nt), b, t0 + mt * 128 + q * 32 + lane, n0, nt);
            mbar_arrive(BAR(B_INIT + (i & 1)));
        };
        if (n_mine > 0) init_tile(0);
        for (int i = 0; i < n_mine; i++) {
            if (i + 1 < n_mine) init_tile(i + 1);
            int b, t0, ntile;
            decode(i, b, t0, ntile);
            const int n0 = ntile * nt;
            const int len = p.lens ? p.lens[b] : p.T;
            mbar_wait_u(BAR(B_ACC + (i & 1)), (i >> 1) & 1);
            for (int mt = 0; mt < MT; mt++)
                acc_tail_tile<8, GEN>(p, acc0 + ((uint32_t)(q * 32) << 16) + (uint32_t)(((i & 1) * MT + mt) * nt), b, t0 + mt * 128 + q * 32 + lane, n0, nt, len);
        }
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------
// The > 48 KB dynamic shared memory opt-in is a per-device (per-context) function attribute: call once per device before
// the first launch there (bv2_engine::finalize does; the kernel test harness calls it itself).
inline void tc_clear_error() {
    const int z = 0;
    BV2_CUDA(cudaMemcpyToSymbol(g_tc_err_dev, &z, sizeof(z)));
}
// Returns the host view of this device's error flag (pinned, host-mapped; raised by a barrier timeout in any wgmma kernel).
inline int* tc_init_device() {
    const int mx = 227 * 1024;
#define BV2_SMEM_ATTR(k) BV2_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, mx))
    BV2_SMEM_ATTR((k_tc_conv1d<0, 0>)); BV2_SMEM_ATTR((k_tc_conv1d<1, 0>)); BV2_SMEM_ATTR((k_tc_conv1d<0, 1>)); BV2_SMEM_ATTR((k_tc_conv1d<1, 1>));
    BV2_SMEM_ATTR((k_tc_conv1d_persist<0, 0>)); BV2_SMEM_ATTR((k_tc_conv1d_persist<1, 0>));
    BV2_SMEM_ATTR((k_tc_conv1d_persist<0, 1>)); BV2_SMEM_ATTR((k_tc_conv1d_persist<1, 1>));
    BV2_SMEM_ATTR((k_tc_conv1d_pstream<0, 0>)); BV2_SMEM_ATTR((k_tc_conv1d_pstream<1, 0>));
    BV2_SMEM_ATTR((k_tc_conv1d_pstream<0, 1>)); BV2_SMEM_ATTR((k_tc_conv1d_pstream<1, 1>));
#undef BV2_SMEM_ATTR
    int* h = nullptr;
    BV2_CUDA(cudaHostAlloc(&h, sizeof(int), cudaHostAllocMapped));
    *h = 0;
    int* d = nullptr;
    BV2_CUDA(cudaHostGetDevicePointer(&d, h, 0));
    BV2_CUDA(cudaMemcpyToSymbol(g_tc_err_flag, &d, sizeof(d)));
    tc_clear_error();
    return h;
}

// Which kernel a tc_conv1d call runs and with what pipeline shape.  tc_conv_plan() is a pure host function of the shapes, the epilogue
// flags and num_sms (no device access), so a test can state which variant a case reaches.
enum TcKind { TC_ONE_TILE = 0, TC_PERSIST = 1, TC_PSTREAM = 2 };
struct TcConvPlan {
    int kind = TC_ONE_TILE;
    int gen = 0, f16 = 0;   // template arguments: generic epilogue, FP16 operands
    int res_smem = 0;       // LayerNorm tail with the residual tile staged in shared memory
    int nas = 0, nws = 0;   // activation / weight ring stages (persist: weights resident, nws = 0)
    size_t smem = 0;        // dynamic shared memory per CTA
    dim3 grid, block;
    int mtiles = 0, ntiles = 0, total = 0;  // persistent kernels: 128-row tiles per batch row, N tiles, tiles in all
};

// x: c4 input [B][x.C/4][T][4]; y: c4 output ([B][y.C/4][T*max(1,ups_u)][4]).  Channel windows via e.cin_off/e.cout_off.
// With e.in_f16 / e.out_f16 the tensor is the 16-bit c8 form [B][C/8][T][8] (Act.p reinterpreted).
// Fills the kernel parameters p and returns the plan; throws on an unsupported combination.
inline TcConvPlan tc_conv_plan(const TcConvW& w, const float* bias, const Act& x, const Act& y, const TcEpi& e, int num_sms, TcParams& p) {
    const int u = w.ups_u ? w.ups_u : 1;
    const int F16 = w.f16;
    BV2_CHECK(w.w && x.B == y.B && y.T == x.T * u, "tc_conv1d shapes");
    BV2_CHECK(e.cin_off % 4 == 0 && e.cout_off % 4 == 0 && e.cin_off + w.Cin <= x.C, "tc_conv1d channel window");
    p = TcParams{};
    TcConvPlan pl;
    pl.f16 = F16;
    p.x = x.p; p.y = y.p; p.w = w.w; p.bias = bias; p.res = e.res; p.bias_b = e.bias_b; p.lens = e.lens;
    p.Cin_total = x.C; p.cin_off = e.cin_off; p.Cout_total = y.C; p.cout_off = e.cout_off;
    p.res_C_total = e.res_C_total ? e.res_C_total : y.C; p.res_c_off = e.res_c_off; p.bias_b_stride = e.bias_b_stride;
    p.T = x.T; p.B = x.B; p.K = w.K; p.dil = e.dil; p.pad = (w.K - 1) / 2 * e.dil;
    p.KC = w.KC; p.nchunks = w.nchunks;
    // Output window: the kernel variant and its pipeline shape are chosen for the whole length (p.T) and only the tiles covering the
    // window are launched, so every output keeps the reduction order of the full-length launch.
    const int t_end = e.t_end < 0 ? y.T : e.t_end;
    BV2_CHECK(0 <= e.t_begin && e.t_begin < t_end && t_end <= y.T && e.t_begin % u == 0 && t_end % u == 0, "tc_conv1d output window");
    p.t_begin = e.t_begin / u; p.t_end = t_end / u;
    const int wrows = p.t_end - p.t_begin;
    const int nt = w.nt;
    if (w.ups_u) BV2_CHECK(w.ups_cout % 4 == 0, "ups cout");
    p.nt = nt;
    const int ntiles = w.Cout / nt;
    const int halo = (w.K - 1) * e.dil;
    p.in_slope = e.in_slope; p.out_scale = e.out_scale; p.accumulate = e.accumulate; p.relu = e.relu; p.res_mode = e.res ? (e.res_mode ? e.res_mode : 1) : 0;
    p.in_mask = e.in_mask; p.out_mask = e.out_mask; p.ups_u = w.ups_u; p.ups_cout = w.ups_cout;
    p.out_tf32 = e.out_tf32; p.skip_xform = e.skip_xform; p.in_f16 = e.in_f16; p.out_f16 = e.out_f16;
    p.ln_gamma = e.ln_gamma; p.ln_beta = e.ln_beta; p.gate = e.gate;
    if (e.gate) BV2_CHECK(F16 && !w.ups_u && !e.res && !e.accumulate && !e.relu && !e.out_f16 && !e.ln_gamma && e.cout_off % 8 == 0 && y.C % 8 == 0 && 2 * y.C >= w.Cout, "gate epilogue");
    if (e.ln_gamma) BV2_CHECK(e.ln_beta && ntiles == 1 && nt % 32 == 0 && !w.ups_u && !e.out_f16 && !e.out_tf32 && !e.relu && e.out_scale == 1.f && e.res_mode != 2 && e.cout_off % 4 == 0, "LayerNorm tail needs one N tile holding every channel");
    if (e.skip_xform) BV2_CHECK(!F16 && w.K == 1 && e.in_slope == 1.f && !e.in_mask, "skip_xform needs a TF32 plain 1x1 conv input");
    if (e.in_f16) BV2_CHECK(F16 && e.in_slope == 1.f && !e.in_mask && e.cin_off % 8 == 0 && x.C % 8 == 0, "in_f16: the 16-bit tensor is the operand image (activation / mask applied by its producer)");
    if (e.out_f16) BV2_CHECK(F16 && !w.ups_u && e.cout_off % 8 == 0 && y.C % 8 == 0 && !e.res && !e.accumulate, "out_f16 epilogue");
    if (p.in_mask || p.out_mask) BV2_CHECK(e.lens != nullptr, "mask needs lens");
    BV2_CHECK(!(p.relu && (p.res_mode || p.accumulate)), "relu cannot be combined with residual/accumulate (accumulator-init fusion)");
    const bool generic = w.ups_u || e.bias_b || e.relu || e.out_f16 || e.ln_gamma || e.gate;
    pl.gen = generic ? 1 : 0;
    const uint32_t esz = F16 ? 2u : 4u;
    p.w_stage_bytes = (uint32_t)(p.KC * nt) * esz;
    auto set_rows = [&](int MT) {
        p.MT = MT; p.R = MT * 128 + halo;
        if (F16 && !e.in_f16) { p.a_op_off = (uint32_t)(p.KC * p.R * 4); p.a_stage_bytes = (uint32_t)(p.KC * p.R * 6); }
        else { p.a_op_off = 0; p.a_stage_bytes = (uint32_t)(p.KC * p.R) * esz; }
    };
    set_rows(1);
    const long long nctas = (long long)cdiv(p.T, 128) * ntiles * p.B;

    // ---- narrow layer with many tiles: persistent CTAs, resident weights, double-buffered accumulator image
    const size_t w_all = (size_t)p.K * p.KC * nt * esz;
    if (!e.skip_xform && !e.in_f16 && !e.out_f16 && !e.ln_gamma && !e.gate && p.nchunks == 1 && ntiles == 1 && w_all <= 64 * 1024 && nctas >= 2 * num_sms) {
        p.nas = 3;
        const size_t wb = (w_all + 127) & ~(size_t)127;
        p.acc_cols = (uint32_t)(2 * nt);
        const size_t smem_p = tc::acc_img_bytes(p.acc_cols) + wb + (size_t)p.nas * p.a_stage_bytes + (size_t)(3 * p.nas + 5) * 8 + 16;
        const int per_sm = 1;  // 512 threads at > 64 registers: one CTA per SM
        const int mtiles = cdiv(wrows, 128);
        const int total = mtiles * p.B;
        const int grid_p = std::min(total, per_sm * num_sms);
        pl.kind = TC_PERSIST; pl.nas = p.nas; pl.nws = 0; pl.smem = smem_p; pl.grid = dim3(grid_p); pl.block = dim3(512);
        pl.mtiles = mtiles; pl.ntiles = 1; pl.total = total;
        return pl;
    }
    // ---- wide layer with at least one tile per SM: persistent CTAs, continuously streamed weights, double-buffered accumulator image
    // (only when two activation and two weight stages fit next to the double-buffered accumulator image; otherwise one tile per CTA)
    if (!e.skip_xform && !e.in_f16 && !e.ln_gamma && nctas >= num_sms && nt >= 64 &&
        tc::acc_img_bytes((uint32_t)(2 * nt)) + 2ull * p.a_stage_bytes + 2ull * p.w_stage_bytes + 2048 <= 220 * 1024) {
        // 128-row tiles: the double-buffered accumulator image (2 x nt columns) already takes up to 132 KB of shared memory
        const int MT = 1;
        set_rows(MT);
        const uint32_t img = tc::acc_img_bytes((uint32_t)(2 * MT * nt));
        const uint32_t big = 220 * 1024 - img;
        int nas2 = std::min(4, std::max(2, p.nchunks * 2));
        while (nas2 > 2 && (size_t)nas2 * p.a_stage_bytes + 3 * (size_t)p.w_stage_bytes + 2048 > big) nas2--;
        int nws2 = (int)((big - (size_t)nas2 * p.a_stage_bytes - 2048) / p.w_stage_bytes);
        nws2 = std::max(2, std::min(nws2, 8));
        p.nas = nas2; p.nws = nws2;
        p.acc_cols = (uint32_t)(2 * MT * nt);
        const size_t smem_s = img + (size_t)nas2 * p.a_stage_bytes + (size_t)nws2 * p.w_stage_bytes + (size_t)(3 * nas2 + 2 * nws2 + 4) * 8 + 16;
        BV2_CHECK(smem_s <= 227 * 1024, "tc_conv1d pstream shared memory");
        const int mtiles = cdiv(wrows, 128 * MT);
        const int total = mtiles * p.B * ntiles;
        const int grid_s = std::min(total, num_sms);
        pl.kind = TC_PSTREAM; pl.nas = p.nas; pl.nws = p.nws; pl.smem = smem_s; pl.grid = dim3(grid_s); pl.block = dim3(512);
        pl.mtiles = mtiles; pl.ntiles = ntiles; pl.total = total;
        return pl;
    }
    // ---- one tile per CTA.  512 threads holding up to 96 fp32 accumulators each: one CTA per SM, so the rings take what the SM has.
    BV2_CHECK(tc_one_tile_nt(nt) && tc_one_tile_nk(p.KC, F16), "tc_conv1d: no one-tile MMA issuer for N tile " + std::to_string(nt) + " / K chunk " +
              std::to_string(p.KC) + " (N tile 16, 32, 48, 64, 96, 128 or 192; K chunk of 1, 2, 4 or (TF32) 8 k-steps)");
    uint32_t budget = 200 * 1024;
    // LayerNorm tail with a residual, at most one CTA per SM (small batches: the launch is a latency chain, not a throughput problem):
    // the residual tile is staged in shared memory by TMA (nt/4 channel groups x 128 rows x 16 B) instead of being pre-loaded into the
    // accumulator; the rings shrink to make room (the weight ring never needs more stages than the conv has)
    const bool res_smem = e.ln_gamma && p.res_mode == 1 && !p.accumulate && nctas <= num_sms && p.res_c_off % 4 == 0 &&
                          tc::acc_img_bytes((uint32_t)nt) + (size_t)nt * 512u + 2ull * p.a_stage_bytes + 2ull * p.w_stage_bytes + 2048 <= 224 * 1024;
    const uint32_t res_bytes = res_smem ? (uint32_t)nt * 512u : 0u;
    const uint32_t img = tc::acc_img_bytes((uint32_t)nt);
    budget = std::min(budget, 224u * 1024u - img);
    if (res_smem) budget = 224 * 1024 - img - res_bytes;
    int nas = std::min(3, std::max(2, p.nchunks));
    while (nas > 2 && (size_t)nas * p.a_stage_bytes + 4 * (size_t)p.w_stage_bytes + 1024 > budget) nas--;
    p.nas = nas;
    int nws = ((int)budget - nas * (int)p.a_stage_bytes - 1024) / (int)p.w_stage_bytes;
    p.nws = std::max(2, std::min(nws, 8));
    p.nws = std::max(2, std::min(p.nws, p.nchunks * p.K));
    p.acc_cols = (uint32_t)nt;
    size_t smem = img + (size_t)p.nas * p.a_stage_bytes + (size_t)p.nws * p.w_stage_bytes + (size_t)(3 * p.nas + 2 * p.nws + 3) * 8 + 16;
    if (res_smem) { smem = (smem + 15) & ~(size_t)15; p.res_soff = (uint32_t)(smem - img); smem += res_bytes; }  // offset from the kernel's `smem` (behind the image)
    BV2_CHECK(smem <= 227 * 1024, "tc_conv1d shared memory");
    pl.kind = TC_ONE_TILE; pl.res_smem = res_smem ? 1 : 0; pl.nas = p.nas; pl.nws = p.nws; pl.smem = smem;
    pl.grid = dim3(cdiv(wrows, 128), ntiles, p.B); pl.block = dim3(512);
    pl.mtiles = cdiv(wrows, 128); pl.ntiles = ntiles; pl.total = pl.mtiles * ntiles * p.B;
    return pl;
}

// Runs the kernel tc_conv_plan() picks.
inline void tc_conv1d(const TcConvW& w, const float* bias, const Act& x, const Act& y, const TcEpi& e, cudaStream_t st, int num_sms) {
    TcParams p;
    const TcConvPlan pl = tc_conv_plan(w, bias, x, y, e, num_sms, p);
    if (pl.kind == TC_PERSIST) {
        if (pl.gen) launch_pdl(pl.f16 ? k_tc_conv1d_persist<1, 1> : k_tc_conv1d_persist<1, 0>, pl.grid, pl.block, pl.smem, st, p, pl.mtiles, pl.total);
        else launch_pdl(pl.f16 ? k_tc_conv1d_persist<0, 1> : k_tc_conv1d_persist<0, 0>, pl.grid, pl.block, pl.smem, st, p, pl.mtiles, pl.total);
    } else if (pl.kind == TC_PSTREAM) {
        if (pl.gen) launch_pdl(pl.f16 ? k_tc_conv1d_pstream<1, 1> : k_tc_conv1d_pstream<1, 0>, pl.grid, pl.block, pl.smem, st, p, pl.mtiles, pl.ntiles, pl.total);
        else launch_pdl(pl.f16 ? k_tc_conv1d_pstream<0, 1> : k_tc_conv1d_pstream<0, 0>, pl.grid, pl.block, pl.smem, st, p, pl.mtiles, pl.ntiles, pl.total);
    } else {
        if (pl.gen) launch_pdl(pl.f16 ? k_tc_conv1d<1, 1> : k_tc_conv1d<1, 0>, pl.grid, pl.block, pl.smem, st, p);
        else launch_pdl(pl.f16 ? k_tc_conv1d<0, 1> : k_tc_conv1d<0, 0>, pl.grid, pl.block, pl.smem, st, p);
    }
}

// TF32 batched GEMMs on c4 operands (attention of the tf32 engine).
inline void tc_launch_simple(TcParams& p, int ntiles, int zdim, cudaStream_t st) {
    const int halo = (p.K - 1) * p.dil;
    p.MT = 1; p.R = 128 + halo; p.pad = (p.K - 1) / 2 * p.dil;
    p.a_stage_bytes = (uint32_t)(p.KC * p.R * 4); p.a_op_off = 0;
    p.w_stage_bytes = (uint32_t)(p.KC * p.nt * 4);
    BV2_CHECK(tc_one_tile_nt(p.nt) && tc_one_tile_nk(p.KC, 0), "tc gemm N tile / K chunk");
    const long long nctas = (long long)cdiv(p.T, 128) * ntiles * zdim;
    const uint32_t img = tc::acc_img_bytes((uint32_t)p.nt);
    const uint32_t budget = std::min<uint32_t>(nctas > 132 ? 100 * 1024 : 200 * 1024, 220 * 1024 - img);
    int nas = std::min(3, std::max(2, p.nchunks));
    while (nas > 2 && (size_t)nas * p.a_stage_bytes + 3 * (size_t)p.w_stage_bytes + 1024 > budget) nas--;
    p.nas = nas;
    int nws = ((int)budget - nas * (int)p.a_stage_bytes - 1024) / (int)p.w_stage_bytes;
    p.nws = std::max(2, std::min(nws, 8));
    p.acc_cols = (uint32_t)p.nt;
    const size_t smem = img + (size_t)p.nas * p.a_stage_bytes + (size_t)p.nws * p.w_stage_bytes + (size_t)(3 * p.nas + 2 * p.nws + 3) * 8 + 16;
    BV2_CHECK(smem <= 227 * 1024, "tc gemm shared memory");
    dim3 grid(cdiv(p.T, 128), ntiles, zdim);
    launch_pdl(k_tc_conv1d<0, 0>, grid, dim3(512), smem, st, p);
}

// S[z][keys][queries] (c4 over keys) = Q . K^T for every (batch, head): qkv c4 [B][3H/4][T][4], q pre-scaled.
// Keys are padded to Fp (multiple of 128); columns >= T hold garbage and are never read by the softmax.
inline void tc_attn_qk(const Act& qkv, int H, int heads, const Act& S, cudaStream_t st) {
    const int dk = H / heads;
    TcParams p{};
    p.x = qkv.p; p.y = S.p; p.w = qkv.p; p.bias = nullptr;
    p.Cin_total = qkv.C; p.cin_off = 0; p.x_c_zstride = dk; p.Cout_total = S.C; p.cout_off = 0; p.res_C_total = S.C;
    p.T = qkv.T; p.B = qkv.B; p.K = 1; p.dil = 1; p.KC = 32; p.nchunks = dk / 32; p.nt = 128;
    p.in_slope = 1.f; p.out_scale = 1.f;
    p.zsplit = heads; p.x_batch_z = 0; p.y_batch_z = 1;
    p.w_mode = 1; p.w_ld = qkv.T; p.w_rows = qkv.T; p.w_c_total = qkv.C; p.w_c_off = H; p.w_c_zstride = dk;
    p.skip_xform = 1;  // q/k/v were rounded to TF32 by the QKV projection's tail
    BV2_CHECK(dk % 32 == 0 && S.C % 128 == 0 && S.T == qkv.T && S.B == qkv.B * heads, "tc_attn_qk shapes");
    tc_launch_simple(p, S.C / 128, qkv.B * heads, st);
}

// att[b][h*dk + d][i] += sum_j P[z][j][i] * V[j][d]  (P = c4 over keys, vt = packed V^T [z][Fp/32][8][dk][4])
inline void tc_attn_pv(const Act& P, const float* vt, int H, int heads, const Act& att, cudaStream_t st) {
    const int dk = H / heads;
    TcParams p{};
    p.x = P.p; p.y = att.p; p.w = vt; p.bias = nullptr;
    p.Cin_total = P.C; p.cin_off = 0; p.Cout_total = att.C; p.cout_off = 0; p.y_c_zstride = dk; p.res_C_total = att.C;
    p.T = P.T; p.B = att.B; p.K = 1; p.dil = 1; p.KC = 64; p.nchunks = P.C / 64; p.nt = dk;  // long reduction (keys): big chunks
    p.in_slope = 1.f; p.out_scale = 1.f; p.accumulate = 1;
    p.zsplit = heads; p.x_batch_z = 1; p.y_batch_z = 0;
    p.w_mode = 0; p.w_zstride = (long long)P.C * dk;
    p.skip_xform = 1;  // P rounded by k_attn_softmax, V^T is a copy of the rounded v
    p.out_tf32 = 1;    // conv_o consumes it without a prologue
    BV2_CHECK(dk % 16 == 0 && dk <= 256 && P.C % 64 == 0 && P.B == att.B * heads && att.T == P.T, "tc_attn_pv shapes");
    tc_launch_simple(p, 1, P.B, st);
}

}  // namespace bv2
