// "G2": the HiFi-GAN Generator (reference models.py:538-557, modules.py:296-309) on 16-bit activation tensors.
//
// Round-2 ncu of the fp32-activation conv family (tc_conv.cuh) showed the MRF convs neither HBM- nor tensor-bound: every staged
// fp32 tile went through a generic-proxy prologue (lrelu + fp32 -> f16 in shared memory, 6 B of smem per element) before the
// MMAs could start, which left room for only ~40 KB of weight stages in flight per SM (Little's law against the ~1.2 us L2
// latency: ~5 TB/s of weight streaming over the whole chip, a third of what the tensor pipe consumes at N = 128).
//
// Here every Generator activation lives in HBM as the MMA operand image itself:
//   H8 tensor  [B][C/8][Tp][8 halves], value = f16(lrelu_0.1(x)), Tp = G2_PADL + T + G2_PADR rows with ZERO halo rows
//   * every consumer of a Generator activation applies lrelu(., 0.1) first (ups, convs1, convs2), so the producer's tail
//     applies it once; the one other use, the residual `x + conv2(..)`, recovers x = a >= 0 ? a : 10 a  (lrelu is invertible);
//     conv_post's lrelu(., 0.01) is a >= 0 ? a : 0.1 a.  CPU simulation of the f16 storage on the oracle: waveform RMS error
//     7.7e-5 (f16 operands, fp32 activations) -> 1.0e-4 (f16 storage), bar 1e-3.
//   * a [KC/8][R rows][16 B] window of such a tensor is the K-major no-swizzle wgmma operand tile: the TMA producer copies it
//     straight into the ring (one cp.async.bulk per channel group), the MMA warp consumes it -- no prologue warps, 2 B of smem
//     per element, and conv zero padding is the tensor's own zero halo (no per-tile fill, no predicates);
//   * tap j of a dilated conv is the same staged tile with the descriptor start advanced by j*dil rows (as in tc_conv.cuh).
//
// One kernel, k_g2_conv: a CTA owns a super-tile of NG x MG m-tiles (128 rows each) x nt <= 128 columns, NG*MG*nt <= 128 columns of
// fp32 accumulator image in shared memory (the whole accumulator of the super-tile), so each weight stage (chunk c, tap j) feeds MG
// 128-row MMAs:
//   streamed weights (C >= 64): NG = 1, MG = 128/nt -- weights cross L2->SM once per MG*128 rows, ring of up to 16 stages;
//   resident weights (C <= 32): all taps loaded once, the M-groups pipeline through the activation ring and the tail of
//   group g overlaps the MMAs of group g+1.
// 640 threads: warp 0 activation producer, warp 2 weight producer, warp 3 output halo, warps 16-19 MMA warpgroup (warp 1 idle),
// warps 4-15 epilogue (accumulator init with the bias before the MMAs; tail accumulator image -> [+ residual] [+ MRF running sum] -> lrelu -> f16
// -> 16-byte coalesced stores).
#pragma once
#include "tc_conv.cuh"

namespace bv2 {

constexpr int G2_PADL = 32, G2_PADR = 32;  // zero halo rows before t = 0 / after t = T-1 (max conv padding: (11-1)/2*5 = 25)

// 16-bit Generator activation; p points at physical row 0 of (b = 0, channel group 0); physical rows [-G2_PADL, Tp - G2_PADL) are
// allocated.  Logical row t (t in [-G2_PADL, T + G2_PADR)) lives at physical row t - base.  A whole tensor has base 0 and
// Tp = G2_PADL + T + G2_PADR; a tensor of a bounded stream (gen_stream.cuh) holds only the rows [base, base + Tp - G2_PADL).
struct H8 {
    uint4* p = nullptr;
    int B = 0, C = 0, T = 0, Tp = 0, base = 0;
    int lim() const { return base + Tp - G2_PADL; }  // logical end of the storage
    // address of logical row 0 of (b = 0, channel group 0): row t of block k is row0()[k * Tp + t] for resident t.  With base > 0 this
    // points before the allocation, so it is computed as an integer address and only ever offset back into the storage.
    uint4* row0() const { return reinterpret_cast<uint4*>(reinterpret_cast<uintptr_t>(p) - (uintptr_t)base * sizeof(uint4)); }
    static size_t bytes(int B, int C, int T) { return (size_t)B * (C / 8) * (size_t)(G2_PADL + T + G2_PADR) * 16; }
};

struct G2Params {
    const uint4* x; uint4* y; const uint4* res; const void* w; const float* bias; const float* bias_b;
    int x_cg, x_Tp, y_cg, y_Tp, res_cg, res_Tp, bias_b_stride;
    int T, K, dil, pad, nt, KC, nchunks, NG, MG, R, nas, nws, resident;
    int t_begin, t_end;  // rows [t_begin, t_end) of the M axis are computed and stored (M = output time; input time of a ConvTranspose)
    uint32_t a_stage_bytes, w_stage_bytes, acc_cols;  // acc_cols: columns of the accumulator image
    int residual, accumulate, ups_u, ups_cout;
    float out_scale;
    int x_lim;  // end of the input rows that may be read: the halo's end T + G2_PADR, or the storage's end if that comes first
};

namespace tc {
__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; e++) { const float2 t = __half22float2(h[e]); f[2 * e] = t.x; f[2 * e + 1] = t.y; }
}
__device__ __forceinline__ float unlrelu10(float a) { return a >= 0.f ? a : a * 10.f; }
}  // namespace tc

// MMAs of one weight stage (chunk c, tap j): MG m-tiles x NK k-steps (NK compile-time), each m-tile one wg_mma over the
// accumulator image.
template <int NK, int MG>
__device__ __forceinline__ void g2_issue_stage(uint32_t d0, uint32_t a_lo0, uint32_t b_lo0, uint32_t a_kstep, uint32_t b_kstep, uint64_t hi, uint32_t nt) {
#pragma unroll 1
    for (int mt = 0; mt < MG; mt++)
        tc::wg_mma<1>(d0 + (uint32_t)mt * nt, hi | (a_lo0 + (uint32_t)(mt * 128)), hi | b_lo0, a_kstep, b_kstep, NK, (int)nt, 1u);
}

// State the MMA issuer carries through its loops (all warp-uniform)
struct G2Issue {
    uint32_t bar_af, bar_ae, bar_wf, bar_we, bar_acc;      // first barrier of each group
    uint32_t a_lo_base, w_lo_base, a_stage16, w_stage16;   // descriptor low words of ring slot 0, slot strides (16-byte units)
    uint32_t a_kstep, b_kstep, nt, dil, tm;
    uint32_t nas, nws;
    int NG, NCH, K, streamed;
    uint64_t hi;
};

// The issuer's loop nest for one (NK, MG) instantiation.  Ring slots, parities, barrier addresses and descriptor words are carried
// incrementally (adds and compares only: no runtime integer division in front of every stage's MMAs).
template <int NK, int MG>
__device__ __forceinline__ void g2_issuer(const G2Issue& q) {
    using namespace tc;
    uint32_t sa = 0, aph = 0, a_cur = q.a_lo_base;   // activation ring slot, parity, descriptor low word of the slot
    uint32_t sw = 0, wph = 0, w_cur = q.w_lo_base;   // weight ring (streamed) / tap cursor (resident)
    uint32_t dg = q.tm;
    for (int g = 0; g < q.NG; g++, dg += (uint32_t)MG * q.nt) {
        if (!q.streamed) w_cur = q.w_lo_base;
        for (int c = 0; c < q.NCH; c++) {
            mbar_wait_u(q.bar_af + 8u * sa, aph);
            uint32_t a_tap = a_cur;
            for (int j = 0; j < q.K; j++, a_tap += q.dil) {
                if (q.streamed) mbar_wait_u(q.bar_wf + 8u * sw, wph);
                g2_issue_stage<NK, MG>(dg, a_tap, w_cur, q.a_kstep, q.b_kstep, q.hi, q.nt);
                if (q.streamed) wg_commit(q.bar_we + 8u * sw);
                w_cur += q.w_stage16;
                if (q.streamed && ++sw == q.nws) { sw = 0; wph ^= 1u; w_cur = q.w_lo_base; }
            }
            wg_commit(q.bar_ae + 8u * sa);
            a_cur += q.a_stage16;
            if (++sa == q.nas) { sa = 0; aph ^= 1u; a_cur = q.a_lo_base; }
        }
        wg_commit(q.bar_acc + 8u * (uint32_t)g);
    }
}
// MG dispatch as a binary tree of two-way branches (a switch would become a jump table: BRX on a vector register makes ptxas treat
// the code after it as divergent and takes the descriptors out of the uniform datapath)
template <int NK>
__device__ __forceinline__ void g2_issuer_mg(const G2Issue& q, int MG) {
    if (MG <= 4) {
        if (MG <= 2) { if (MG == 1) g2_issuer<NK, 1>(q); else g2_issuer<NK, 2>(q); }
        else { if (MG == 3) g2_issuer<NK, 3>(q); else g2_issuer<NK, 4>(q); }
    } else {
        if (MG <= 6) { if (MG == 5) g2_issuer<NK, 5>(q); else g2_issuer<NK, 6>(q); }
        else { if (MG == 7) g2_issuer<NK, 7>(q); else g2_issuer<NK, 8>(q); }
    }
}

__global__ void __launch_bounds__(640, 1) k_g2_conv(G2Params p) {
    using namespace tc;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + acc_img_bytes(p.acc_cols);  // behind the accumulator image
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;  // shfl: warp-uniform for the compiler
    const int NAS = p.nas, NWS = p.nws, NG = p.NG, MG = p.MG, NCH = p.nchunks, nt = p.nt, R = p.R;
    const int t0 = p.t_begin + blockIdx.x * NG * MG * 128, ntile = blockIdx.y, n0 = ntile * nt, b = blockIdx.z;
    uint8_t* sA = smem;
    uint8_t* sW = smem + (size_t)NAS * p.a_stage_bytes;
    const int nwst = p.resident ? NCH * p.K : NWS;  // weight stages held in shared memory
    uint64_t* bars = reinterpret_cast<uint64_t*>(sW + (size_t)nwst * p.w_stage_bytes);
    const uint32_t bar0 = smem_u32(bars);
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
    // barrier map: a_full[NAS], a_empty[NAS], w_full[NWS], w_empty[NWS], acc_full[NG], acc_init
    const int B_AFULL = 0, B_AEMPTY = NAS, B_WFULL = 2 * NAS, B_WEMPTY = 2 * NAS + NWS, B_ACC = 2 * NAS + 2 * NWS, B_INIT = B_ACC + NG;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NAS; i++) { mbar_init(BAR(B_AFULL + i), 1); mbar_init(BAR(B_AEMPTY + i), 1); }
        for (int i = 0; i < NWS; i++) { mbar_init(BAR(B_WFULL + i), 1); mbar_init(BAR(B_WEMPTY + i), 1); }
        for (int i = 0; i < NG; i++) mbar_init(BAR(B_ACC + i), 1);
        mbar_init(BAR(B_INIT), 12 * 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const uint32_t acc0 = 0;  // accumulator image base (acc_ptr)
    const int ncg = p.KC / 8;  // 16-byte channel groups per chunk

    if (warp == 0) {
        // ===== activation producer (reads the upstream kernel's output: PDL wait first)
        asm volatile("griddepcontrol.wait;" ::: "memory");
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        const int steps = NG * NCH;
        for (int s = 0; s < steps; s++) {
            const int g = s / NCH, c = s - g * NCH, sa = s % NAS;
            const int row0 = t0 + g * MG * 128 - p.pad;
            const int nrows = max(0, min(R, p.x_lim - row0));  // never read past the tensor's halo or storage; rows beyond (and rows past a window's end) feed discarded outputs only
            if (lane == 0) {
                mbar_wait(BAR(B_AEMPTY + sa), ((s / NAS) & 1) ^ 1);
                mbar_expect_tx(BAR(B_AFULL + sa), (uint32_t)nrows * 16u * (uint32_t)ncg);
            }
            __syncwarp();
            if (lane < ncg && nrows > 0) {
                const uint4* src = p.x + ((size_t)b * p.x_cg + (size_t)c * ncg + lane) * p.x_Tp + row0;
                bulk_g2s(smem_u32(sA + (size_t)sa * p.a_stage_bytes) + (uint32_t)lane * (uint32_t)R * 16u, src, (uint32_t)nrows * 16u, BAR(B_AFULL + sa));
            }
        }
    } else if (warp == 2) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        if (lane == 0) {
            // ===== weight producer (weights do not depend on the upstream kernel: no PDL wait)
            const uint8_t* wt = reinterpret_cast<const uint8_t*>(p.w) + (size_t)ntile * NCH * p.K * p.w_stage_bytes;
            if (p.resident) {
                const uint32_t total = (uint32_t)(NCH * p.K) * p.w_stage_bytes;
                mbar_expect_tx(BAR(B_WFULL), total);
                for (uint32_t off = 0; off < total; off += 32768u)
                    bulk_g2s(smem_u32(sW) + off, wt + off, min(32768u, total - off), BAR(B_WFULL));
            } else {
                // slot / parity / addresses carried incrementally (the producer has to out-run the MMA issuer: no division, no call)
                const uint32_t bar_wf = BAR(B_WFULL), bar_we = BAR(B_WEMPTY), dst0 = smem_u32(sW), nws_u = (uint32_t)NWS;
                uint32_t sw = 0, ph = 1u, dst = dst0;
                for (int g = 0; g < NG; g++) {
                    const uint8_t* src = wt;
                    for (int cj = 0; cj < NCH * p.K; cj++, src += p.w_stage_bytes) {
                        mbar_wait_u(bar_we + 8u * sw, ph);
                        mbar_expect_tx(bar_wf + 8u * sw, p.w_stage_bytes);
                        bulk_g2s(dst, src, p.w_stage_bytes, bar_wf + 8u * sw);
                        dst += p.w_stage_bytes;
                        if (++sw == nws_u) { sw = 0; ph ^= 1u; dst = dst0; }
                    }
                }
            }
        }
    } else if (warp >= 16) {
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        // ===== MMA warpgroup (warps 16-19): all 128 threads run the loops together (wgmma is warpgroup-collective)
        // Descriptors are kept as (constant high word, 32-bit low word): start address >> 4 in bits [0,14), LBO >> 4 in [16,30) of the low
        // word; tap / m-tile / k-step offsets are plain 32-bit adds on the low word (shared memory addresses stay below 2^18), which the
        // compiler keeps in the uniform datapath.
        const uint32_t a_lo_c = (((uint32_t)R * 16u) >> 4) << 16, b_lo_c = (((uint32_t)nt * 16u) >> 4) << 16;
        const uint32_t desc_hi = 128u >> 4;  // SBO = 128 B
        const uint32_t a_kstep = 2u * (uint32_t)R, b_kstep = 2u * (uint32_t)nt;
        const uint32_t tm = acc0;
        const int nk = p.KC / 16;
        if (p.resident) mbar_wait_u(BAR(B_WFULL), 0);
        mbar_wait_u(BAR(B_INIT), 0);  // accumulators hold the bias: every MMA accumulates
        G2Issue q;
        q.bar_af = BAR(B_AFULL); q.bar_ae = BAR(B_AEMPTY); q.bar_wf = BAR(B_WFULL); q.bar_we = BAR(B_WEMPTY); q.bar_acc = BAR(B_ACC);
        q.a_lo_base = ((smem_u32(sA) & 0x3ffffu) >> 4) | a_lo_c; q.w_lo_base = ((smem_u32(sW) & 0x3ffffu) >> 4) | b_lo_c;
        q.a_stage16 = p.a_stage_bytes >> 4; q.w_stage16 = p.w_stage_bytes >> 4;
        q.a_kstep = a_kstep; q.b_kstep = b_kstep; q.nt = (uint32_t)nt; q.dil = (uint32_t)p.dil; q.tm = tm;
        q.nas = (uint32_t)NAS; q.nws = (uint32_t)NWS; q.NG = NG; q.NCH = NCH; q.K = p.K;
        q.streamed = !p.resident;
        q.hi = (uint64_t)desc_hi << 32;
        if (nk == 2) g2_issuer_mg<2>(q, MG);
        else g2_issuer_mg<1>(q, MG);  // g2_conv() admits KC = 16 or 32 only
    } else if (warp == 3) {
        // ===== zero halo of the OUTPUT tensor (= the conv padding of its consumers), written by its producer: the CTA of the first super-tile
        // clears rows [-G2_PADL, 0) if the window starts at t = 0, the CTA of the last one rows [T_out, T_out + G2_PADR) if the window ends at
        // T_out, for every channel group of batch b (N tile 0 only).  A window inside the tensor leaves the halo rows alone: in a streamed run
        // they are final rows of earlier windows.
        const bool lo = blockIdx.x == 0 && p.t_begin == 0, hi = blockIdx.x == gridDim.x - 1 && p.t_end == p.T;
        if (ntile == 0 && (lo || hi)) {
            asm volatile("griddepcontrol.wait;" ::: "memory");  // the rows may alias a tensor an upstream kernel is still reading
            uint4* yb = p.y + (size_t)b * p.y_cg * p.y_Tp;
            const int Tout = p.T * (p.ups_u ? p.ups_u : 1);
            const uint4 z4 = make_uint4(0u, 0u, 0u, 0u);
            if (lo)
                for (int i = lane; i < p.y_cg * G2_PADL; i += 32) yb[(size_t)(i / G2_PADL) * p.y_Tp + (i % G2_PADL) - G2_PADL] = z4;
            if (hi)
                for (int i = lane; i < p.y_cg * G2_PADR; i += 32) yb[(size_t)(i / G2_PADR) * p.y_Tp + Tout + (i % G2_PADR)] = z4;
        }
    } else if (warp >= 4 && warp < 16) {
        // ===== epilogue, 12 warps: row quarter q = warp & 3; the 3 warps of a quarter share the (m-tile, 32-column batch) items
        // round-robin.  Two phases:
        //   init (before the MMAs, before the PDL wait: touches only static data and the CTA-private accumulator image): the accumulators are pre-loaded
        //        with bias (+ per-batch bias) by image stores, so every MMA accumulates and the tail has no bias loads / adds;
        //   tail: the accumulator image -> [+ residual] [+ MRF running sum] -> lrelu -> f16 -> coalesced 16-byte stores.
        // The tail is instruction-bound (two-three warps per scheduler cannot hide ALU latency: round-2 ncu), so it is kept lean.
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
        const int e = warp - 4, q = warp & 3, part = e >> 2;
        const uint32_t trow = acc0 + ((uint32_t)(q * 32) << 16);
        const int u = p.ups_u;
        const int ncb = nt >= 32 ? nt / 32 : 1, cw = nt >= 32 ? 32 : 16;  // column batches per m-tile, columns per batch
        {
            for (int cb = part; cb < ncb; cb += 3) {
                const int col0 = cb * cw;
                uint32_t v[32];
#pragma unroll
                for (int h = 0; h < 8; h++) {
                    if (4 * h < cw) {
                        const int n = n0 + col0 + 4 * h;
                        float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + (u ? n % p.ups_cout : n)));
                        if (p.bias_b) {
                            const float4 c4 = __ldg(reinterpret_cast<const float4*>(p.bias_b + (size_t)b * p.bias_b_stride + n));
                            b4.x += c4.x; b4.y += c4.y; b4.z += c4.z; b4.w += c4.w;
                        }
                        v[4 * h] = __float_as_uint(b4.x); v[4 * h + 1] = __float_as_uint(b4.y); v[4 * h + 2] = __float_as_uint(b4.z); v[4 * h + 3] = __float_as_uint(b4.w);
                    }
                }
                for (int m = 0; m < NG * MG; m++) {
                    if (cw == 32) acc_st<32>(trow + (uint32_t)(m * nt + col0), v); else acc_st<16>(trow + (uint32_t)(m * nt + col0), v);
                }
            }
            mbar_arrive(BAR(B_INIT));
        }
        asm volatile("griddepcontrol.wait;" ::: "memory");
        const bool scaled = p.out_scale != 1.f;
        for (int g = 0; g < NG; g++) {
            mbar_wait(BAR(B_ACC + g), 0);
            for (int it = part; it < MG * ncb; it += 3) {
                const int mt = it / ncb, col0 = (it - mt * ncb) * cw;
                const int t = t0 + (g * MG + mt) * 128 + q * 32 + lane;
                const bool ok = t < p.t_end;  // stores, residual reads and running-sum updates stay inside the window
                uint32_t v[32];
                if (cw == 32) acc_ld<32>(trow + (uint32_t)((g * MG + mt) * nt + col0), v); else acc_ld<16>(trow + (uint32_t)((g * MG + mt) * nt + col0), v);
                // residual / running-sum operands are fetched while the accumulator image load is in flight
                uint4 r4[4], a4[4];
                size_t yo[4];
#pragma unroll
                for (int h = 0; h < 4; h++) {
                    if (8 * h < cw) {
                        const int n = n0 + col0 + 8 * h;  // first of 8 consecutive output columns
                        if (u) { const int r = n / p.ups_cout, co = n - r * p.ups_cout; yo[h] = ((size_t)b * p.y_cg + co / 8) * p.y_Tp + (size_t)t * u + r; }
                        else yo[h] = ((size_t)b * p.y_cg + n / 8) * p.y_Tp + t;
                        if (p.residual && ok) r4[h] = p.res[((size_t)b * p.res_cg + n / 8) * p.res_Tp + t];
                        if (p.accumulate && ok) a4[h] = p.y[yo[h]];
                    }
                }
                if (!ok) continue;
#pragma unroll
                for (int h = 0; h < 4; h++) {
                    if (8 * h < cw) {
                        float f[8];
#pragma unroll
                        for (int k = 0; k < 8; k++) f[k] = __uint_as_float(v[8 * h + k]);
                        if (p.residual) {
                            float r8[8];
                            unpack8(r4[h], r8);
#pragma unroll
                            for (int k = 0; k < 8; k++) f[k] += unlrelu10(r8[k]);
                        }
                        if (p.accumulate) {
                            float a8[8];
                            unpack8(a4[h], a8);
#pragma unroll
                            for (int k = 0; k < 8; k++) f[k] += unlrelu10(a8[k]);
                        }
                        if (scaled) {
#pragma unroll
                            for (int k = 0; k < 8; k++) f[k] *= p.out_scale;
                        }
#pragma unroll
                        for (int k = 0; k < 8; k++) f[k] = fmaxf(f[k], 0.1f * f[k]);  // lrelu(x, 0.1) = max(x, 0.1 x)
                        uint4 o;
                        o.x = pack_h2(f[0], f[1]); o.y = pack_h2(f[2], f[3]); o.z = pack_h2(f[4], f[5]); o.w = pack_h2(f[6], f[7]);
                        p.y[yo[h]] = o;
                    }
                }
            }
        }
    }
    __syncthreads();
}

// fp32 c4 [B][C/4][T][4] (rows t >= lens[b] read as zero) -> raw f16 H8 (no activation): the Generator's input z * y_mask, rows
// [t_begin, t_end) of it, into an H8 whose physical row 0 is logical row y_base
__global__ void __launch_bounds__(128) k_c4_to_h8(const float4* __restrict__ x, uint4* __restrict__ y, int C, int T, int Tp, const int* __restrict__ lens,
                                                  int t_begin, int t_end, int y_base) {
    const int t = t_begin + blockIdx.x * blockDim.x + threadIdx.x, g = blockIdx.y, b = blockIdx.z;
    // zero halo of the output (conv_pre's padding): first / last block of each channel-group run, when the window reaches that end
    if (blockIdx.x == 0 && t_begin == 0 && threadIdx.x < G2_PADL) y[((size_t)b * (C / 8) + g) * Tp + (int)threadIdx.x - G2_PADL] = make_uint4(0u, 0u, 0u, 0u);
    if (blockIdx.x == gridDim.x - 1 && t_end == T && threadIdx.x < G2_PADR) y[((size_t)b * (C / 8) + g) * Tp + (T - y_base) + threadIdx.x] = make_uint4(0u, 0u, 0u, 0u);
    if (t >= t_end) return;
    const bool in = !lens || t < lens[b];
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), c = a;
    if (in) { a = x[((size_t)b * (C / 4) + 2 * g) * T + t]; c = x[((size_t)b * (C / 4) + 2 * g + 1) * T + t]; }
    uint4 o;
    o.x = tc::pack_h2(a.x, a.y); o.y = tc::pack_h2(a.z, a.w); o.z = tc::pack_h2(c.x, c.y); o.w = tc::pack_h2(c.z, c.w);
    y[((size_t)b * (C / 8) + g) * Tp + (t - y_base)] = o;
}

// conv_post (C -> 1, K taps, no bias) + tanh on an H8 input (reference models.py:553-555: F.leaky_relu default slope 0.01,
// recovered from the stored lrelu_0.1 value as a >= 0 ? a : 0.1 a); the zero halo supplies the conv padding.
// The kernel is issue-bound, not HBM-bound (17 MB at config 2): with one output per thread reading its own K rows every element was
// unpacked + activated K times and every FMA fetched its weight from shared memory (~40 instructions per 16-byte load, 24 us).  Here a block
// stages TB + K - 1 rows ONCE as activated fp32 in shared memory (coalesced 16-byte loads, conflict-free stores), the weights ride in the
// kernel parameters (constant bank: FFMA takes them as an operand), and a thread's inner loop is one conflict-free LDS + one FFMA per tap.
template <int C, int K> struct PostW { float w[C * K]; };  // [C][K]
// Outputs [t_begin, t_end) of the T samples are stored; staged rows past t_end feed discarded outputs only.  x holds the logical rows
// from x_base (H8::base; 0 for a whole tensor) to the end of its storage; rows from the halo's end T + G2_PADR on, or from the storage's
// end if that comes first, are read as zero.
template <int C, int K>
__global__ void __launch_bounds__(256) k_conv_post_tanh_h8(const uint4* __restrict__ x, int Tp, int x_base, const __grid_constant__ PostW<C, K> pw,
                                                           float* __restrict__ y, int T, int t_begin, int t_end) {
    constexpr int TB = 512, RW = TB + K - 1, LD = RW + 2;  // outputs per block, staged rows, row stride of the staged tile
    __shared__ float sx[C][LD];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    const int t0 = t_begin + blockIdx.x * TB, b = blockIdx.y, row_end = min(T + G2_PADR, x_base + Tp - G2_PADL);
    for (int i = threadIdx.x; i < (C / 8) * RW; i += blockDim.x) {
        const int g = i / RW, r = i - g * RW, row = t0 - K / 2 + r;  // row >= -K/2 >= -G2_PADL
        float f[8];
        if (row < row_end) tc::unpack8(x[((size_t)b * (C / 8) + g) * Tp + (row - x_base)], f);
        else {
#pragma unroll
            for (int k = 0; k < 8; k++) f[k] = 0.f;
        }
#pragma unroll
        for (int k = 0; k < 8; k++) sx[g * 8 + k][r] = fmaxf(f[k], 0.1f * f[k]);  // a >= 0 ? a : 0.1 a
    }
    __syncthreads();
#pragma unroll
    for (int o = 0; o < TB / 256; o++) {
        const int tl = threadIdx.x + o * 256, t = t0 + tl;
        float acc = 0.f;
#pragma unroll
        for (int g = 0; g < C / 8; g++) {
#pragma unroll
            for (int j = 0; j < K; j++) {
#pragma unroll
                for (int k = 0; k < 8; k++) acc = fmaf(sx[g * 8 + k][tl + j], pw.w[(g * 8 + k) * K + j], acc);
            }
        }
        if (t < t_end) y[(size_t)b * T + t] = tanhf(acc);
    }
}

// Slide of a bounded stream (gen_stream_slides): for each descriptor, rows [src, src + rows) of every one of its `blocks` row blocks
// (B x C/8, row stride Tp) move to [dst, dst + rows).  Source and destination never overlap (dst + rows <= src), so the copy has no
// order.  16-byte vectors; blockIdx.y picks the descriptor.
struct G2SlideDesc { uint4* p; int blocks, Tp, src, dst, rows; };  // p: physical row 0 of row block 0 (H8::p)
constexpr int G2_SLIDE_MAX = 120;  // descriptors per launch: the parameter block stays below 4 KB
struct G2SlideParams { int n; G2SlideDesc d[G2_SLIDE_MAX]; };
__global__ void __launch_bounds__(256) k_g2_slide(const __grid_constant__ G2SlideParams sp) {
    asm volatile("griddepcontrol.wait;" ::: "memory");  // the rows were written by the kernels before this one
    const G2SlideDesc& d = sp.d[blockIdx.y];
    const long long n = (long long)d.blocks * d.rows;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int blk = (int)(i / d.rows), r = (int)(i - (long long)blk * d.rows);
        uint4* row0 = d.p + (size_t)blk * d.Tp;
        row0[d.dst + r] = row0[d.src + r];
    }
}

inline void g2_init_device() {
    BV2_CUDA(cudaFuncSetAttribute(k_g2_conv, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
}

struct G2Epi {
    const H8* res = nullptr;  // y = lrelu(conv + bias + unlrelu(res))
    int accumulate = 0;       // ... + unlrelu(y_old)   (MRF running sum)
    float out_scale = 1.f;
    const float* bias_b = nullptr; int bias_b_stride = 0;  // per-batch bias (speaker conditioning of conv_pre)
    int dil = 1;
    int t_begin = 0, t_end = -1;  // output window [t_begin, t_end) (t_end = -1: T_out); a ConvTranspose window is a multiple of its stride
    int st_override = 0;      // tests: force the super-tile size (m-tiles per CTA)
};

// Static part of the plan (fixed at weight-pack time): N tile and K chunk for a conv with `cols` output columns.
inline int g2_nt(int cols) { int nt = std::min(cols, 128); while (cols % nt || nt % 16) nt -= 16; return nt; }
inline int g2_kc(int Cin) { return Cin >= 128 ? 32 : 16; }

// Launch shape of a g2_conv call.  g2_conv_plan() is a pure host function of the shapes and num_sms (no device access), so a test can
// state which variant a case reaches.
struct G2Plan {
    int resident = 0;       // all weight taps loaded once (else streamed through a ring of nws stages)
    int NG = 1, MG = 1;     // super-tile: NG groups of MG 128-row m-tiles per CTA
    int nas = 0, nws = 0;   // activation / weight ring stages
    size_t smem = 0;        // dynamic shared memory per CTA
    dim3 grid;
};

// x: H8 input, y: H8 output (T_out = T * max(1, ups_u)).  w packed by tc_pack_weights / tc_pack_upsample with f16 = 1, nt = g2_nt, kc = g2_kc.
// Fills the kernel parameters p and returns the plan; throws on an unsupported combination.
inline G2Plan g2_conv_plan(const TcConvW& w, const float* bias, const H8& x, const H8& y, const G2Epi& e, int num_sms, G2Params& p) {
    const int u = w.ups_u ? w.ups_u : 1;
    BV2_CHECK(w.w && w.f16 && bias && x.B == y.B && y.T == x.T * u && x.C == w.Cin && (w.ups_u ? y.C == w.ups_cout : y.C == w.Cout), "g2_conv shapes");
    BV2_CHECK(w.nt <= 128 && (w.KC == 16 || w.KC == 32) && x.C % 8 == 0 && y.C % 8 == 0, "g2_conv tiling (K chunk of 16 or 32 channels)");
    p = G2Params{};
    // x, y and res are addressed by logical row: the pointers are H8::row0(), which only resident rows are read or written through
    p.x = x.row0(); p.y = y.row0(); p.w = w.w; p.bias = bias; p.bias_b = e.bias_b; p.bias_b_stride = e.bias_b_stride;
    p.x_cg = x.C / 8; p.x_Tp = x.Tp; p.y_cg = y.C / 8; p.y_Tp = y.Tp;
    p.x_lim = std::min(x.T + G2_PADR, x.lim());
    if (e.res) {
        BV2_CHECK(!w.ups_u && e.res->C == y.C && e.res->T == y.T && e.res->B == y.B, "g2_conv residual");
        p.res = e.res->row0(); p.res_cg = e.res->C / 8; p.res_Tp = e.res->Tp; p.residual = 1;
    }
    p.accumulate = e.accumulate; p.out_scale = e.out_scale; p.ups_u = w.ups_u; p.ups_cout = w.ups_cout;
    if (w.ups_u) BV2_CHECK(w.ups_cout % 8 == 0 && !e.accumulate, "g2_conv ups");
    p.T = x.T; p.K = w.K; p.dil = e.dil; p.pad = (w.K - 1) / 2 * e.dil;
    BV2_CHECK(p.pad <= G2_PADL && p.pad <= G2_PADR, "g2_conv padding exceeds the tensor halo");
    p.nt = w.nt; p.KC = w.KC; p.nchunks = w.nchunks;
    const int t_end = e.t_end < 0 ? y.T : e.t_end;
    BV2_CHECK(0 <= e.t_begin && e.t_begin < t_end && t_end <= y.T && e.t_begin % u == 0 && t_end % u == 0, "g2_conv output window");
    p.t_begin = e.t_begin / u; p.t_end = t_end / u;
    // every row the window reads or writes is resident (a whole tensor, base 0, always passes)
    BV2_CHECK((x.base == 0 || p.t_begin - p.pad >= x.base) && std::min(p.t_end + p.pad, x.T + G2_PADR) <= x.lim(), "g2_conv input rows not resident");
    BV2_CHECK((y.base == 0 || e.t_begin >= y.base) && (t_end < y.T ? t_end : y.T + G2_PADR) <= y.lim(), "g2_conv output rows not resident");
    if (e.res) BV2_CHECK(e.t_begin >= e.res->base && t_end <= e.res->lim(), "g2_conv residual rows not resident");
    const int ntiles = w.Cout / w.nt, halo = (w.K - 1) * e.dil;
    p.w_stage_bytes = (uint32_t)(w.KC * w.nt * 2);
    // the accumulator image of a CTA holds at most 128 columns of 128 rows (66 KB of shared memory).  The time tiling follows the window;
    // the reduction order of every output (bias, then chunk c, tap j, k-step) does not depend on it.
    const int mtiles = cdiv(p.t_end - p.t_begin, 128), mgmax = std::max(1, 128 / w.nt);
    const size_t img = tc::acc_img_bytes((uint32_t)(mgmax * w.nt)), budget = 220 * 1024 - img;
    const size_t w_all = (size_t)w.nchunks * w.K * p.w_stage_bytes;
    p.resident = w_all <= 48 * 1024 && ntiles == 1;
    // ---- super-tile (m-tiles per CTA): as few CTAs as fill the SMs once; streamed weights want >= 2 m-tiles per weight pass
    int ST = (int)std::min<long long>(mgmax, std::max<long long>(1, ((long long)mtiles * ntiles * x.B + num_sms - 1) / num_sms));
    if (!p.resident && ST < 2 && mgmax >= 2 && mtiles >= 2 && w_all > 256 * 1024) ST = 2;
    if (e.st_override) ST = std::min(e.st_override, mgmax);
    ST = std::min(ST, mtiles);
    int NG = 1, MG = ST;
    auto a_bytes = [&](int mg) { return (size_t)(w.KC / 8) * (size_t)(mg * 128 + halo) * 16; };
    if (p.resident) {
        // pipeline the m-groups through the activation ring: prefer 4 groups, then 2 (whatever wastes the fewest m-tiles)
        int best_ng = 1, best_mg = ST; long long best_cost = -1;
        for (int ng : {4, 2, 1}) {
            const int mg = cdiv(ST, ng);
            if (ng * mg > mgmax || ng > ST || mg > 8) continue;  // the issuer is instantiated for MG <= 8
            const long long ctas = (long long)cdiv(mtiles, ng * mg) * x.B;
            const long long waves = (ctas + num_sms - 1) / num_sms;
            const long long cost = waves * ng * mg;  // m-tile slots per SM
            if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_ng = ng; best_mg = mg; }
        }
        NG = best_ng; MG = best_mg;
    } else {
        while (MG > 1 && 2 * a_bytes(MG) + 4 * (size_t)p.w_stage_bytes + 1024 > budget) MG--;
    }
    MG = std::min(MG, 8);
    p.NG = NG; p.MG = MG; p.R = MG * 128 + halo;
    p.a_stage_bytes = (uint32_t)a_bytes(MG);
    const int a_steps = NG * w.nchunks;
    size_t wres = p.resident ? w_all : 0;
    int nas = std::min(a_steps, p.resident ? 4 : 3);
    while (nas > 2 && (size_t)nas * p.a_stage_bytes + wres + (p.resident ? 0 : 8 * (size_t)p.w_stage_bytes) + 1024 > budget) nas--;
    nas = std::max(1, nas);
    p.nas = nas;
    if (p.resident) p.nws = 1;
    else p.nws = (int)std::max<size_t>(2, std::min<size_t>(16, (budget - (size_t)nas * p.a_stage_bytes - 1024) / p.w_stage_bytes));
    if (!p.resident) p.nws = std::min(p.nws, NG * w.nchunks * w.K);
    p.acc_cols = (uint32_t)(NG * MG * w.nt);
    const size_t smem = tc::acc_img_bytes(p.acc_cols) + (size_t)nas * p.a_stage_bytes + (p.resident ? w_all : (size_t)p.nws * p.w_stage_bytes) + (size_t)(2 * nas + 2 * p.nws + NG + 3) * 8 + 16;
    BV2_CHECK(smem <= 227 * 1024, "g2_conv shared memory");
    G2Plan pl;
    pl.resident = p.resident; pl.NG = NG; pl.MG = MG; pl.nas = nas; pl.nws = p.nws; pl.smem = smem;
    pl.grid = dim3(cdiv(mtiles, NG * MG), ntiles, x.B);
    return pl;
}

inline void g2_conv(const TcConvW& w, const float* bias, const H8& x, const H8& y, const G2Epi& e, cudaStream_t st, int num_sms) {
    G2Params p;
    const G2Plan pl = g2_conv_plan(w, bias, x, y, e, num_sms, p);
    launch_pdl(k_g2_conv, pl.grid, dim3(640), pl.smem, st, p);
}

}  // namespace bv2
