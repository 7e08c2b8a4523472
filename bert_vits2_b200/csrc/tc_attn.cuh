// Fused windowed relative-position multi-head self-attention of the flow's transformer layers on Hopper wgmma
// (reference attentions.py:263-322 via attentions.py:103-120, called 16x per infer by TransformerCouplingBlock, models.py:82-145):
//     scores[i,j] = q_i.k_j + [|j-i| <= w] q_i.Ek[j-i+w]      (q pre-scaled by 1/sqrt(dk) in the QKV projection weights)
//     p = softmax_j(scores, keys j >= len excluded)            out_i = sum_j p_ij v_j + sum_r p_{i,i+r-w} Ev[r]
// One CTA = 128 queries of one (batch, head), split over two consumer warpgroups of 64 query rows each.  S = Q.K^T of a key tile
// is a register accumulator of the warpgroup (wgmma, both operands in shared memory); the softmax runs on that fragment and the
// probabilities go to the P.V wgmma straight from registers (the accumulator fragment of S for 16 key columns is the A-operand
// fragment of one k-step), so neither S nor P is ever stored; O = P.V accumulates in registers across the key tiles.
//
// Operands are the 16-bit c8 tensors the QKV projection's epilogue writes ([B][3H/8][T][8 halves]):
//   * a [dk/8][rows][8] tile of q or k IS the K-major no-swizzle operand image (TMA copies it straight from global memory);
//   * v needs no transposition either: [dk/8][keys][8] is the MN-major no-swizzle image of the [keys x dk] B operand
//     (8 keys x 16 bytes = one 128-byte core matrix; LBO = stride between 8-key blocks, SBO = stride between 8-channel blocks).
// Two passes over the key tiles instead of an online softmax: pass A computes the row maxima (Q.K^T + max only), pass B
// recomputes Q.K^T, exponentiates against the final maximum and feeds P.V -- no accumulator rescaling.
//
// Key split (B = 1 leaves only 2 heads x F/128 query tiles = 16 CTAs for 132 SMs, each walking every key tile twice): a cluster of
// ks CTAs shares a query tile, CTA r handles key tiles r, r + ks, ... with its OWN running maximum, and the partial results
// (m_r, l_r, relative-value weights, unnormalised P.V rows) are merged flash-decoding style over distributed shared memory:
//     m = max_r m_r,  w_r = 2^((m_r - m) log2 e),  out = (sum_r w_r O_r + sum_r w_r prel_r . Ev) / sum_r w_r l_r
// Each CTA parks its partial rows in its own shared memory (the K/V stages are free by then), one cluster barrier, CTA c pulls
// rows [c*128/ks, (c+1)*128/ks) of every peer (ld.shared::cluster) in fixed rank order -- deterministic -- and writes them.
// Without a key split (ks = 1) the same merge runs on the CTA's own rows.
// 288 threads: warps 0-7 = two consumer warpgroups (scores, softmax, P.V, parking, merge), warp 8 = TMA producer (Q once, K tiles
// twice, V tiles once).
#pragma once
#include "tc_conv.cuh"

namespace bv2 {

struct AttnParams {
    const uint4* qkv;   // 16-bit c8 [B][3H/8][T][8]: q | k | v channel blocks of H each, head h at channels h*dk
    uint4* att;         // 16-bit c8 [B][H/8][T][8]
    const float* rel_k; const float* rel_v;  // [2w+1][dk]
    const int* lens;    // valid length per batch (keys >= len excluded, query rows >= len produce zeros)
    int B, T, H, heads, window;
    int ks;             // key split: a cluster of ks CTAs shares one 128-query tile, CTA r takes key tiles r, r + ks, ... (1 = no cluster)
    uint32_t v_lbo, v_sbo;  // MN-major descriptor strides of the V operand
};

namespace tc {
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ void unpack_h8(const uint4& u, float* f) {
    const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
    for (int e = 0; e < 4; e++) { const float2 t = __half22float2(h[e]); f[2 * e] = t.x; f[2 * e + 1] = t.y; }
}
}  // namespace tc

// Merge of the key splits (flash-decoding style) for one thread: row m of the query tile, 96/KSC channels.  Every distributed-shared-memory
// load is issued before the first dependent instruction (interleaved with the arithmetic, the 36 loads of a 4-way merge would each
// pay a full distributed-shared-memory round trip one after the other).
// Peers are combined in fixed rank order: deterministic.
template <int KSC, int DK>
__device__ __forceinline__ void attn_merge_rows(uint32_t sK_addr, const float* sEv, int rk, int t, int q0, int len, int T, int nrel, uint4* obase) {
    using namespace tc;
    constexpr int NREL = 9, rows_per = 128 / KSC, nf4 = (DK / 4) / KSC;  // float4 slots (4 channels each) of this thread: 12 (KSC = 2) or 6 (KSC = 4)
    constexpr float LOG2E = 1.4426950408889634f;
    static_assert(DK == 96 && nf4 % 2 == 0, "channel split of the merge");
    const int m = rk * rows_per + t % rows_per, part = t / rows_per, i = q0 + m;
    const uint32_t local = sK_addr + (uint32_t)m * 16u;
    float4 st4[KSC][3], ov[KSC][nf4];
#pragma unroll
    for (int r2 = 0; r2 < KSC; r2++) {
        uint32_t remote;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(r2));
#pragma unroll
        for (int k = 0; k < 3; k++)
            asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(st4[r2][k].x), "=f"(st4[r2][k].y), "=f"(st4[r2][k].z), "=f"(st4[r2][k].w) : "r"(remote + (24u + (uint32_t)k) * 2048u));
        const uint32_t rbase = remote + (uint32_t)(part * nf4) * 2048u;
#pragma unroll
        for (int g = 0; g < nf4; g++)
            asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(ov[r2][g].x), "=f"(ov[r2][g].y), "=f"(ov[r2][g].z), "=f"(ov[r2][g].w) : "r"(rbase + (uint32_t)g * 2048u));
    }
    float M = -INFINITY;
#pragma unroll
    for (int r2 = 0; r2 < KSC; r2++) M = fmaxf(M, st4[r2][0].x);
    float L = 0.f;
    float prel[NREL];
#pragma unroll
    for (int r = 0; r < NREL; r++) prel[r] = 0.f;
    float o[4 * nf4];
#pragma unroll
    for (int e = 0; e < 4 * nf4; e++) o[e] = 0.f;
#pragma unroll
    for (int r2 = 0; r2 < KSC; r2++) {
        const float4 a4 = st4[r2][0], b4 = st4[r2][1], c4 = st4[r2][2];  // (m, l, prel0, prel1), prel2..5, prel6..8
        const float wgt = a4.x == -INFINITY ? 0.f : ex2_approx((a4.x - M) * LOG2E);
        L = fmaf(wgt, a4.y, L);
        prel[0] = fmaf(wgt, a4.z, prel[0]); prel[1] = fmaf(wgt, a4.w, prel[1]);
        prel[2] = fmaf(wgt, b4.x, prel[2]); prel[3] = fmaf(wgt, b4.y, prel[3]); prel[4] = fmaf(wgt, b4.z, prel[4]); prel[5] = fmaf(wgt, b4.w, prel[5]);
        prel[6] = fmaf(wgt, c4.x, prel[6]); prel[7] = fmaf(wgt, c4.y, prel[7]); prel[8] = fmaf(wgt, c4.z, prel[8]);
#pragma unroll
        for (int g = 0; g < nf4; g++) {
            const float4 v4 = ov[r2][g];
            o[4 * g] = fmaf(wgt, v4.x, o[4 * g]); o[4 * g + 1] = fmaf(wgt, v4.y, o[4 * g + 1]);
            o[4 * g + 2] = fmaf(wgt, v4.z, o[4 * g + 2]); o[4 * g + 3] = fmaf(wgt, v4.w, o[4 * g + 3]);
        }
    }
    const float inv = (i < len && L > 0.f) ? 1.f / L : 0.f;
    const int ch0 = part * nf4 * 4;  // first channel of this thread
#pragma unroll
    for (int r = 0; r < NREL; r++) {
        if (r < nrel) {
            const float pw = prel[r];
            const float* ev = &sEv[r * DK + ch0];
#pragma unroll
            for (int e = 0; e < 4 * nf4; e++) o[e] = fmaf(pw, ev[e], o[e]);
        }
    }
    if (i < T) {
#pragma unroll
        for (int g = 0; g < nf4 / 2; g++) {
            uint4 u;
            u.x = pack_h2(o[8 * g] * inv, o[8 * g + 1] * inv); u.y = pack_h2(o[8 * g + 2] * inv, o[8 * g + 3] * inv);
            u.z = pack_h2(o[8 * g + 4] * inv, o[8 * g + 5] * inv); u.w = pack_h2(o[8 * g + 6] * inv, o[8 * g + 7] * inv);
            obase[(size_t)(ch0 / 8 + g) * T + i] = u;
        }
    }
}

template <int DK, int KT>
__global__ void __launch_bounds__(288, 1) k_flow_attn(AttnParams p) {
    using namespace tc;
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int NG = DK / 8, NREL = 9;
    constexpr uint32_t QB = DK * 128 * 2, KB = DK * KT * 2;
    constexpr float LOG2E = 1.4426950408889634f;
    static_assert(KT == 128 && DK == 96, "tile shape (wgmma_ss_n128 / wgmma_rs_n96_tb)");
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + QB;
    uint8_t* sV = sK + 2 * KB;
    float* sEk = reinterpret_cast<float*>(sV + 2 * KB);
    float* sEv = sEk + NREL * DK;
    float* sQrel = sEv + NREL * DK;    // [NREL][128 rows]: q_i . Ek[r] of this CTA's query rows
    float* sPrel = sQrel + NREL * 128; // [NREL][128 rows]: p[i, i + r - w], written by the pass-B thread that meets that key
    uint64_t* bars = reinterpret_cast<uint64_t*>(sPrel + NREL * 128);
    const uint32_t bar0 = smem_u32(bars);
    auto BAR = [&](int i) { return bar0 + 8u * (uint32_t)i; };
    enum { B_QFULL = 0, B_KFULL = 1, B_KEMPTY = 3, B_VFULL = 5, B_VEMPTY = 7, NBARS = 9 };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int KS = p.ks, rk = (int)blockIdx.x % KS;  // cluster dims (KS,1,1): rank in cluster == blockIdx.x % KS
    const int q0 = ((int)blockIdx.x / KS) * 128, h = blockIdx.y, b = blockIdx.z;
    const int H8 = p.H / 8;
    const int w = p.window, nrel = 2 * w + 1;

    if (threadIdx.x == 0) {
        mbar_init(BAR(B_QFULL), 1);
        for (int i = 0; i < 2; i++) { mbar_init(BAR(B_KFULL + i), 1); mbar_init(BAR(B_KEMPTY + i), 2); mbar_init(BAR(B_VFULL + i), 1); mbar_init(BAR(B_VEMPTY + i), 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // V tiles are loaded with partial row counts at the end of the sequence: rows never written must hold finite values (they meet
    // p = 0 in the P.V MMA), so both V stages start zeroed; later partial loads leave finite rows of an earlier tile behind.
    for (int i = threadIdx.x; i < (int)(2 * KB / 16); i += blockDim.x) reinterpret_cast<uint4*>(sV)[i] = make_uint4(0u, 0u, 0u, 0u);
    for (int i = threadIdx.x; i < nrel * DK; i += blockDim.x) { sEk[i] = p.rel_k[i]; sEv[i] = p.rel_v[i]; }
    fence_async_smem();
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    const int len = min(p.lens ? p.lens[b] : p.T, p.T);
    const int NT_all = q0 < len ? (len + KT - 1) / KT : 0;  // key tiles that hold at least one valid key (same for the whole cluster)
    const int NT = NT_all > rk ? (NT_all - rk + KS - 1) / KS : 0;  // ... of which this CTA takes tiles rk, rk + KS, ...
    const uint4* qbase = p.qkv + ((size_t)b * 3 * H8 + (size_t)h * NG) * p.T;
    const uint4* kbase = qbase + (size_t)H8 * p.T;
    const uint4* vbase = kbase + (size_t)H8 * p.T;
    uint4* obase = p.att + ((size_t)b * H8 + (size_t)h * NG) * p.T;

    if (warp == 8) {
        if (NT > 0) {
            const int nq = min(128, p.T - q0);
            if (lane == 0) mbar_expect_tx(BAR(B_QFULL), (uint32_t)nq * 16u * NG);
            __syncwarp();
            if (lane < NG) bulk_g2s(smem_u32(sQ) + (uint32_t)lane * 128u * 16u, qbase + (size_t)lane * p.T + q0, (uint32_t)nq * 16u, BAR(B_QFULL));
            for (int s = 0; s < 2 * NT; s++) {
                const int j = s < NT ? s : s - NT, k0 = (rk + KS * j) * KT, nk = min(KT, p.T - k0), st = s & 1;
                if (lane == 0) {
                    mbar_wait(BAR(B_KEMPTY + st), ((s >> 1) & 1) ^ 1);
                    mbar_expect_tx(BAR(B_KFULL + st), (uint32_t)nk * 16u * NG);
                }
                __syncwarp();
                if (lane < NG)
                    bulk_g2s(smem_u32(sK) + (uint32_t)st * KB + (uint32_t)lane * KT * 16u, kbase + (size_t)lane * p.T + k0, (uint32_t)nk * 16u, BAR(B_KFULL + st));
                if (s >= NT) {
                    const int vs = j & 1;
                    if (lane == 0) {
                        mbar_wait(BAR(B_VEMPTY + vs), ((j >> 1) & 1) ^ 1);
                        mbar_expect_tx(BAR(B_VFULL + vs), (uint32_t)nk * 16u * NG);
                    }
                    __syncwarp();
                    if (lane < NG)
                        bulk_g2s(smem_u32(sV) + (uint32_t)vs * KB + (uint32_t)lane * KT * 16u, vbase + (size_t)lane * p.T + k0, (uint32_t)nk * 16u, BAR(B_VFULL + vs));
                }
            }
        }
    } else if (NT_all == 0) {  // every query of this tile is padding: zeros (written once per cluster)
        const int i = q0 + (int)threadIdx.x;
        if (threadIdx.x < 128 && i < p.T && rk == 0)
            for (int g = 0; g < NG; g++) obase[(size_t)g * p.T + i] = make_uint4(0u, 0u, 0u, 0u);
    } else {
        // consumer warpgroup wg owns query rows [64 wg, 64 wg + 64); this thread holds rows r0 and r0 + 8 of the wgmma fragments
        // and, in each 8-column block, columns cq and cq + 1
        const int ct = threadIdx.x, wg = ct >> 7, t = ct & 127;
        const int r0 = 64 * wg + 16 * (t >> 5) + ((t & 31) >> 2), cq = 2 * (t & 3);
        float M[2] = {-INFINITY, -INFINITY}, L[2] = {0.f, 0.f};
        float o[DK / 2];
#pragma unroll
        for (int e = 0; e < DK / 2; e++) o[e] = 0.f;
        if (NT > 0) {
            mbar_wait(BAR(B_QFULL), 0);
            if (ct < 128) {
                // ---- relative-key logits of row m: qrel[r] = q_i . Ek[r]
                const int m = ct;
                float qrel[NREL];
#pragma unroll
                for (int r = 0; r < NREL; r++) qrel[r] = 0.f;
                for (int g = 0; g < NG; g++) {
                    float qf[8];
                    unpack_h8(reinterpret_cast<const uint4*>(sQ)[g * 128 + m], qf);
#pragma unroll
                    for (int r = 0; r < NREL; r++) {
                        if (r < nrel) {
                            const float4 e0 = *reinterpret_cast<const float4*>(&sEk[r * DK + g * 8]), e1 = *reinterpret_cast<const float4*>(&sEk[r * DK + g * 8 + 4]);
                            float a = qrel[r];  // same accumulation order as a scalar loop over the 8 channels
                            a = fmaf(qf[0], e0.x, a); a = fmaf(qf[1], e0.y, a); a = fmaf(qf[2], e0.z, a); a = fmaf(qf[3], e0.w, a);
                            a = fmaf(qf[4], e1.x, a); a = fmaf(qf[5], e1.y, a); a = fmaf(qf[6], e1.z, a); a = fmaf(qf[7], e1.w, a);
                            qrel[r] = a;
                        }
                    }
                }
#pragma unroll
                for (int r = 0; r < NREL; r++) { sQrel[r * 128 + m] = qrel[r]; sPrel[r * 128 + m] = 0.f; }
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");  // both consumer warpgroups: the qrel / prel tables are complete
            const uint64_t qd = make_desc(smem_u32(sQ), 128u * 16u, 128u) + (uint64_t)(64 * wg);  // 64 rows further = 8 core-matrix groups
            // S (64 rows x KT keys of this warpgroup) = Q . K_tile^T, then the K stage goes back to the producer
            auto scores = [&](int s, float* c) {
                const int st = s & 1;
                mbar_wait(BAR(B_KFULL + st), (s >> 1) & 1);
#pragma unroll
                for (int e = 0; e < KT / 2; e++) c[e] = 0.f;
                const uint64_t kd = make_desc(smem_u32(sK) + (uint32_t)st * KB, (uint32_t)KT * 16u, 128u);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < DK / 16; kk++) wgmma_ss_n128(c, qd + (uint64_t)(kk * 2 * 128), kd + (uint64_t)(kk * 2 * KT));
                wgmma_commit();
                wgmma_wait0();
                asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
                if (t == 0) mbar_arrive(BAR(B_KEMPTY + st));
            };
            // ---- pass A: row maxima over the valid keys (of this CTA's key tiles)
            for (int s = 0; s < NT; s++) {
                const int k0 = (rk + KS * s) * KT, nvalid = len - k0;
                const bool band = (k0 <= q0 + 127 + w) && (k0 + KT - 1 >= q0 - w);
                float c[KT / 2];
                scores(s, c);
#pragma unroll
                for (int e = 0; e < KT / 2; e++) {
                    const int hr = (e >> 1) & 1, row = r0 + 8 * hr, col = 8 * (e >> 2) + cq + (e & 1);
                    float x = c[e];
                    if (band) { const int d = k0 + col - (q0 + row) + w; if ((unsigned)d < (unsigned)nrel) x += sQrel[d * 128 + row]; }
                    if (col < nvalid) M[hr] = fmaxf(M[hr], x);
                }
            }
#pragma unroll
            for (int hr = 0; hr < 2; hr++) {
                M[hr] = fmaxf(M[hr], __shfl_xor_sync(0xffffffffu, M[hr], 1));
                M[hr] = fmaxf(M[hr], __shfl_xor_sync(0xffffffffu, M[hr], 2));
            }
            // ---- pass B: p = exp(s - M) in registers -> P.V; row sums; relative-value weights
            const float M2[2] = {M[0] * LOG2E, M[1] * LOG2E};
            for (int j = 0; j < NT; j++) {
                const int vs = j & 1, k0 = (rk + KS * j) * KT, nvalid = len - k0;
                const bool band = (k0 <= q0 + 127 + w) && (k0 + KT - 1 >= q0 - w);
                float c[KT / 2];
                scores(NT + j, c);
#pragma unroll
                for (int e = 0; e < KT / 2; e++) {
                    const int hr = (e >> 1) & 1, row = r0 + 8 * hr, col = 8 * (e >> 2) + cq + (e & 1);
                    float x = c[e];
                    int d = -1;
                    if (band) { d = k0 + col - (q0 + row) + w; if ((unsigned)d < (unsigned)nrel) x += sQrel[d * 128 + row]; else d = -1; }
                    const float pe = col < nvalid ? ex2_approx(fmaf(x, LOG2E, -M2[hr])) : 0.f;
                    if (d >= 0) sPrel[d * 128 + row] = pe;  // key j = i + d - w is met exactly once
                    L[hr] += pe;
                    c[e] = pe;
                }
                // the S fragment of key columns [16 kk, 16 kk + 16) is the A fragment of k-step kk
                uint32_t a[KT / 16][4];
#pragma unroll
                for (int kk = 0; kk < KT / 16; kk++) {
                    a[kk][0] = pack_h2(c[8 * kk], c[8 * kk + 1]); a[kk][1] = pack_h2(c[8 * kk + 2], c[8 * kk + 3]);
                    a[kk][2] = pack_h2(c[8 * kk + 4], c[8 * kk + 5]); a[kk][3] = pack_h2(c[8 * kk + 6], c[8 * kk + 7]);
                }
                mbar_wait(BAR(B_VFULL + vs), (j >> 1) & 1);
                const uint64_t vd = make_desc(smem_u32(sV) + (uint32_t)vs * KB, p.v_lbo, p.v_sbo);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < KT / 16; kk++) wgmma_rs_n96_tb(o, a[kk], vd + (uint64_t)(16 * kk));  // 16 keys = two 128-byte key blocks
                wgmma_commit();
                wgmma_wait0();
                asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
                if (t == 0) mbar_arrive(BAR(B_VEMPTY + vs));
            }
#pragma unroll
            for (int hr = 0; hr < 2; hr++) {
                L[hr] += __shfl_xor_sync(0xffffffffu, L[hr], 1);
                L[hr] += __shfl_xor_sync(0xffffffffu, L[hr], 2);
            }
        }
        // ---- park this CTA's partial rows in its own shared memory (the K/V stages, free once both warpgroups are done):
        //      [27 float4][128 rows]: slots 0..23 unnormalised P.V (96 channels), 24 = (m, l, prel0, prel1), 25 = prel2..5, 26 = prel6..8
        asm volatile("bar.sync 1, 256;" ::: "memory");
        float* partf = reinterpret_cast<float*>(sK);
#pragma unroll
        for (int e = 0; e < DK / 2; e += 2) {
            const int hr = (e >> 1) & 1, row = r0 + 8 * hr, ch = 8 * (e >> 2) + cq;
            *reinterpret_cast<float2*>(&partf[((size_t)(ch >> 2) * 128 + row) * 4 + (ch & 3)]) = make_float2(o[e], o[e + 1]);
        }
        __syncwarp();  // sPrel entries of this warp's rows were written by the lanes of their quads
        if ((t & 3) == 0) {
            float4* part = reinterpret_cast<float4*>(sK);
#pragma unroll
            for (int hr = 0; hr < 2; hr++) {
                const int row = r0 + 8 * hr;
                float pr[NREL];
#pragma unroll
                for (int r = 0; r < NREL; r++) pr[r] = NT > 0 ? sPrel[r * 128 + row] : 0.f;
                part[(size_t)24 * 128 + row] = make_float4(M[hr], L[hr], pr[0], pr[1]);
                part[(size_t)25 * 128 + row] = make_float4(pr[2], pr[3], pr[4], pr[5]);
                part[(size_t)26 * 128 + row] = make_float4(pr[6], pr[7], pr[8], 0.f);
            }
        }
    }
    if (NT_all > 0) {
        // ---- merge the key splits (every thread of every CTA of the cluster takes part in both barriers)
        asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
        // CTA rk merges rows [rk * 128/KS, (rk + 1) * 128/KS); KS threads share a row (96/KS channels each), consecutive threads take
        // consecutive rows (coalesced distributed-shared-memory reads)
        if (threadIdx.x < 128) {
            if (KS == 4) attn_merge_rows<4, DK>(smem_u32(sK), sEv, rk, threadIdx.x, q0, len, p.T, nrel, obase);
            else if (KS == 2) attn_merge_rows<2, DK>(smem_u32(sK), sEv, rk, threadIdx.x, q0, len, p.T, nrel, obase);
            else attn_merge_rows<1, DK>(smem_u32(sK), sEv, rk, threadIdx.x, q0, len, p.T, nrel, obase);
        }
        asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");  // peers are done reading this CTA's rows
    }
}

inline size_t tc_flow_attn_smem(int DK, int KT) { return (size_t)DK * 128 * 2 + 4 * (size_t)DK * KT * 2 + 2 * 9 * (size_t)DK * 4 + 2 * 9 * 128 * 4 + 9 * 8 + 16; }

inline void tc_flow_attn_init_device() {
    BV2_CUDA(cudaFuncSetAttribute(k_flow_attn<96, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
}

// qkv16: 16-bit c8 tensor with C = 3H channels (Act.p reinterpreted); att16: 16-bit c8 tensor with C = H channels.
inline void tc_flow_attn(const Act& qkv16, const Act& att16, const float* rel_k, const float* rel_v, const int* lens, int heads, int window,
                         cudaStream_t st, int num_sms, int ks_override = 0) {
    const int H = att16.C, dk = H / heads, KT = 128;
    BV2_CHECK(qkv16.C == 3 * H && dk == 96 && H % 8 == 0 && window <= 4 && qkv16.T == att16.T && qkv16.B == att16.B, "tc_flow_attn shapes (head dim 96, window <= 4)");
    AttnParams p{};
    p.qkv = reinterpret_cast<const uint4*>(qkv16.p); p.att = reinterpret_cast<uint4*>(att16.p);
    p.rel_k = rel_k; p.rel_v = rel_v; p.lens = lens;
    p.B = qkv16.B; p.T = qkv16.T; p.H = H; p.heads = heads; p.window = window;
    p.v_lbo = 128u;                 // MN-major V: stride between 8-key core-matrix blocks (K direction)
    p.v_sbo = (uint32_t)KT * 16u;   // ... and between 8-channel blocks (N direction)
    // key split: as many CTAs per query tile as keep the grid within one wave of the SMs and leave each CTA at least one key tile
    const int qtiles = cdiv(p.T, 128), ctas = qtiles * heads * p.B;
    int ks = 1;
    while (ks < 4 && 2 * ks <= qtiles && ctas * 2 * ks <= num_sms) ks *= 2;  // the merge is written for 2 or 4 splits
    if (ks_override > 0) ks = ks_override;
    p.ks = ks;
    launch_pdl_cluster(k_flow_attn<96, 128>, dim3(qtiles * ks, heads, p.B), dim3(288), tc_flow_attn_smem(dk, KT), st, ks, p);
}

}  // namespace bv2
