// Fused FP32 kernels of the token-rate stage (text encoder, SDP, DP: everything that feeds ceil(durations) stays on FP32 FMA,
// SURVEY.md section 7 H1).  At T ~ 256 tokens this stage is pure launch / dependency latency (~110 small launches unfused),
// so the kernels here trade launches for on-chip fusion: a whole layer per launch, weights staged in shared memory by TMA.
#pragma once
#include "kernels_simt.cuh"
#include "tc_conv.cuh"

namespace bv2 {

// ------------------------------------------------------------------------------------------------
// One DDSConv layer in one launch (reference modules.py:118-130, channels C = 192):
//     y = convs_sep[i](x * x_mask)   depthwise k=3, dilation d      y = gelu(norms_1[i](y))
//     y = convs_1x1[i](y)            dense C x C                    y = gelu(norms_2[i](y))
//     x = x + y                      (* x_mask after the last layer, modules.py:130)
// One CTA = 16 time steps x all channels, 8 warps.  The 1x1 weight matrix (C*C*4 = 144 KB, packed [ci][co]) is staged in
// shared memory with ONE bulk TMA copy that overlaps the depthwise conv + first LayerNorm; both LayerNorms are warp-shuffle
// reductions (one warp owns a time step: phase 1 by channel group, phase 3 by the 6 output channels a lane computed).
// x is read with a halo of +-d from neighbouring tiles, so the layer writes to a different buffer than it reads.
// ------------------------------------------------------------------------------------------------
struct DdsArgs {
    const float* x; float* y;            // c4 [B][C/4][T][4], in / out (different buffers)
    const float* dw_w; const float* dw_b;  // depthwise [C][3], [C]
    const float* w1; const float* b1;      // 1x1 packed [C][C] (ci major, co fastest), bias [C]
    const float* g1; const float* be1; const float* g2; const float* be2;  // LayerNorm gamma / beta
    const int* lens;
    int T, B, dil, last;                 // last: multiply the result by x_mask
};

template <int C>
__global__ void __launch_bounds__(256, 1) k_dds_layer(DdsArgs a) {
    using namespace tc;
    static_assert(C == 192, "lane -> channel mapping below is written for 192 channels (48 c4 groups)");
    constexpr int TT = 16, NCG = C / 4;
    extern __shared__ __align__(128) uint8_t smem[];
    float* sW = reinterpret_cast<float*>(smem);                      // [C][C]
    float* sY = sW + C * C;                                          // [TT][C]: activations between LN1/GELU and the 1x1 conv
    uint64_t* bar = reinterpret_cast<uint64_t*>(sY + C * TT);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t0 = blockIdx.x * TT, b = blockIdx.y;
    if (threadIdx.x == 0) {
        mbar_init(smem_u32(bar), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(smem_u32(bar), (uint32_t)(C * C * 4));
        bulk_g2s(smem_u32(sW), a.w1, (uint32_t)(C * C * 4), smem_u32(bar));  // weights: independent of the upstream kernel
    }
    pdl_wait();
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int len = a.lens ? a.lens[b] : a.T;
    const float4* x4 = reinterpret_cast<const float4*>(a.x) + (size_t)b * NCG * a.T;
    // ---- phase 1: depthwise conv + LayerNorm 1 + GELU; warp w owns time steps 2w, 2w+1; lane owns c4 groups lane and 32+lane (<16)
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const int tt = 2 * warp + k, t = t0 + tt;
        float4 v[2];
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < 2; q++) {
            const int cg = lane + 32 * q;
            v[q] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (cg < NCG && t < a.T) {
                float4 acc = *reinterpret_cast<const float4*>(a.dw_b + cg * 4);
                const float* wc = a.dw_w + cg * 12;
#pragma unroll
                for (int j = 0; j < 3; j++) {
                    const int u = t + (j - 1) * a.dil;
                    if (u >= 0 && u < a.T && u < len) {
                        const float4 xv = x4[(size_t)cg * a.T + u];
                        acc.x = fmaf(xv.x, wc[j], acc.x); acc.y = fmaf(xv.y, wc[3 + j], acc.y);
                        acc.z = fmaf(xv.z, wc[6 + j], acc.z); acc.w = fmaf(xv.w, wc[9 + j], acc.w);
                    }
                }
                v[q] = acc;
                s += (acc.x + acc.y) + (acc.z + acc.w);
            }
        }
        s = warp_sum(s);
        const float mean = s / (float)C;
        float qv = 0.f;
#pragma unroll
        for (int q = 0; q < 2; q++)
            if (lane + 32 * q < NCG) {
                const float dx = v[q].x - mean, dy = v[q].y - mean, dz = v[q].z - mean, dw = v[q].w - mean;
                qv += (dx * dx + dy * dy) + (dz * dz + dw * dw);
            }
        qv = warp_sum(qv);
        const float rstd = rsqrtf(qv / (float)C + 1e-5f);
#pragma unroll
        for (int q = 0; q < 2; q++) {
            const int cg = lane + 32 * q;
            if (cg < NCG) {
                const float4 g = *reinterpret_cast<const float4*>(a.g1 + cg * 4), be = *reinterpret_cast<const float4*>(a.be1 + cg * 4);
                float4 o;
                o.x = gelu_erf((v[q].x - mean) * rstd * g.x + be.x); o.y = gelu_erf((v[q].y - mean) * rstd * g.y + be.y);
                o.z = gelu_erf((v[q].z - mean) * rstd * g.z + be.z); o.w = gelu_erf((v[q].w - mean) * rstd * g.w + be.w);
                *reinterpret_cast<float4*>(&sY[tt * C + cg * 4]) = o;  // consecutive lanes -> consecutive 16 bytes
            }
        }
    }
    __syncthreads();
    mbar_wait(smem_u32(bar), 0);
    // ---- phase 2: 1x1 conv.  warp w: time steps 2w, 2w+1; lane: output channels 4*lane..4*lane+3 and 128+2*lane, 129+2*lane
    float acc[2][6];
    {
        const float4 bA = *reinterpret_cast<const float4*>(a.b1 + 4 * lane);
        const float2 bB = *reinterpret_cast<const float2*>(a.b1 + 128 + 2 * lane);
#pragma unroll
        for (int k = 0; k < 2; k++) { acc[k][0] = bA.x; acc[k][1] = bA.y; acc[k][2] = bA.z; acc[k][3] = bA.w; acc[k][4] = bB.x; acc[k][5] = bB.y; }
    }
    for (int c0 = 0; c0 < C; c0 += 4) {
        // 4 input channels per step: the two time steps' activations are warp-uniform (broadcast) 16-byte loads
        const float4 ya = *reinterpret_cast<const float4*>(&sY[(2 * warp) * C + c0]), yb = *reinterpret_cast<const float4*>(&sY[(2 * warp + 1) * C + c0]);
        const float y0[4] = {ya.x, ya.y, ya.z, ya.w}, y1[4] = {yb.x, yb.y, yb.z, yb.w};
#pragma unroll
        for (int e = 0; e < 4; e++) {  // ascending ci: the summation order is fixed
            const float4 wA = *reinterpret_cast<const float4*>(&sW[(c0 + e) * C + 4 * lane]);
            const float2 wB = *reinterpret_cast<const float2*>(&sW[(c0 + e) * C + 128 + 2 * lane]);
            acc[0][0] = fmaf(y0[e], wA.x, acc[0][0]); acc[0][1] = fmaf(y0[e], wA.y, acc[0][1]); acc[0][2] = fmaf(y0[e], wA.z, acc[0][2]);
            acc[0][3] = fmaf(y0[e], wA.w, acc[0][3]); acc[0][4] = fmaf(y0[e], wB.x, acc[0][4]); acc[0][5] = fmaf(y0[e], wB.y, acc[0][5]);
            acc[1][0] = fmaf(y1[e], wA.x, acc[1][0]); acc[1][1] = fmaf(y1[e], wA.y, acc[1][1]); acc[1][2] = fmaf(y1[e], wA.z, acc[1][2]);
            acc[1][3] = fmaf(y1[e], wA.w, acc[1][3]); acc[1][4] = fmaf(y1[e], wB.x, acc[1][4]); acc[1][5] = fmaf(y1[e], wB.y, acc[1][5]);
        }
    }
    // ---- phase 3: LayerNorm 2 + GELU + residual (+ mask), straight from the accumulators
    const float4 gA = *reinterpret_cast<const float4*>(a.g2 + 4 * lane), eA = *reinterpret_cast<const float4*>(a.be2 + 4 * lane);
    const float2 gB = *reinterpret_cast<const float2*>(a.g2 + 128 + 2 * lane), eB = *reinterpret_cast<const float2*>(a.be2 + 128 + 2 * lane);
    float4* y4 = reinterpret_cast<float4*>(a.y) + (size_t)b * NCG * a.T;
#pragma unroll
    for (int k = 0; k < 2; k++) {
        const int t = t0 + 2 * warp + k;
        float s = ((acc[k][0] + acc[k][1]) + (acc[k][2] + acc[k][3])) + (acc[k][4] + acc[k][5]);
        s = warp_sum(s);
        const float mean = s / (float)C;
        float qv = 0.f;
#pragma unroll
        for (int e = 0; e < 6; e++) { const float d = acc[k][e] - mean; qv += d * d; }
        qv = warp_sum(qv);
        const float rstd = rsqrtf(qv / (float)C + 1e-5f);
        if (t >= a.T) continue;
        const float m = (a.last && t >= len) ? 0.f : 1.f;
        const float4 rA = x4[(size_t)lane * a.T + t];
        float4 oA;
        oA.x = (rA.x + gelu_erf((acc[k][0] - mean) * rstd * gA.x + eA.x)) * m;
        oA.y = (rA.y + gelu_erf((acc[k][1] - mean) * rstd * gA.y + eA.y)) * m;
        oA.z = (rA.z + gelu_erf((acc[k][2] - mean) * rstd * gA.z + eA.z)) * m;
        oA.w = (rA.w + gelu_erf((acc[k][3] - mean) * rstd * gA.w + eA.w)) * m;
        y4[(size_t)lane * a.T + t] = oA;
        // channels 128 + 2*lane, +1 = half of c4 group 32 + lane/2
        const float2* xr = reinterpret_cast<const float2*>(x4 + (size_t)(32 + (lane >> 1)) * a.T + t) + (lane & 1);
        const float2 rB = *xr;
        float2 oB;
        oB.x = (rB.x + gelu_erf((acc[k][4] - mean) * rstd * gB.x + eB.x)) * m;
        oB.y = (rB.y + gelu_erf((acc[k][5] - mean) * rstd * gB.y + eB.y)) * m;
        *(reinterpret_cast<float2*>(y4 + (size_t)(32 + (lane >> 1)) * a.T + t) + (lane & 1)) = oB;
    }
}

inline size_t dds_layer_smem(int C) { return (size_t)C * C * 4 + (size_t)C * 16 * 4 + 16; }
inline void launch_dds_layer(const DdsArgs& a, int C, cudaStream_t st) {
    BV2_CHECK(C == 192, "fused DDS layer is instantiated for 192 channels");
    launch_pdl(k_dds_layer<192>, dim3(cdiv(a.T, 16), a.B), dim3(256), dds_layer_smem(C), st, a);
}


// ------------------------------------------------------------------------------------------------
// Token-rate FP32 GEMM-style Conv1d (K = 1 or 3 taps, dilation 1) with cluster split-K and fused epilogues: replaces
// k_conv1d_c4 + k_layernorm_c4 pairs of the text encoder / duration predictors (reference attentions.py:103-120 conv_o + norm,
// FFN conv_1 / conv_2 + norm attentions.py:438-464; models.py:285-299).
//   one CTA      = 16 time steps x one 192-channel column block x one slice of the input channels (4 warps; warp w owns time
//                  steps 4w..4w+3, lane owns output channels 4*lane..+3 and 128+2*lane,+1: 24 accumulators, every weight load
//                  feeds 4 time steps)
//   weights      streamed through a 3-stage shared-memory ring by bulk TMA copies (16 input channels x K taps x 192 columns per
//                stage), the input tile staged once ([time][ci], zero padding / x_mask applied while staging)
//   split-K      at T = 256 tokens a 768->192 conv has only 16 such tiles; the reduction is therefore cut across a thread-block
//                CLUSTER of `ksplit` CTAs (one per input-channel slice, so each SM streams 1/ksplit of the weights) and the partial
//                tiles are summed through distributed shared memory in fixed rank order (deterministic: ceil(durations) must not
//                depend on scheduling); each rank finishes 16/ksplit rows, so bias / relu / residual + LayerNorm / mask run in the
//                same kernel on rows that hold all 192 channels.
// ------------------------------------------------------------------------------------------------
struct TokGemmArgs {
    const float* x; int Cin_total, cin_off, Cin;   // c4 input [B][Cin_total/4][T][4], channels [cin_off, cin_off + Cin)
    const float* w; int Cout_w;                    // packed [Cin][K][Cout_w] (co fastest)
    const float* bias; const float* bias_b; int bias_b_stride;  // [Cout]; optional per-batch bias row
    float* y; int Cout_total, cout_off;            // c4 output; column block n covers channels cout_off + 192 n ..
    const float* res; int res_C_total;             // LayerNorm mode: y = LN(res + conv) (res: c4, 192 channels at offset 0)
    const float* gamma; const float* beta;         // null: no LayerNorm
    const int* lens;
    // plain-layout input (BERT ingest, reference models.py:386-388): input channel ci comes from plain[ci / plain_C] laid out [B][plain_C][T]
    // (the three 1024-channel feature tensors of get_text are consumed as the caller passes them: no c4 staging copies)
    const float* plain[3]; int plain_C;
    int T, B, relu, in_mask, out_mask, mask_pre, ksplit;  // mask_pre: (conv + bias) * x_mask BEFORE the residual add (FFN: norm(x + ffn(x) * mask))
};

template <int K>
__global__ void __launch_bounds__(128, 1) k_tok_gemm(TokGemmArgs a) {
    using namespace tc;
    constexpr int TT = 16, NB = 192, CK = 16, NST = 3, TTP = TT + K - 1, PAD = (K - 1) / 2;
    extern __shared__ __align__(128) uint8_t smem[];
    const int S = a.ksplit;
    const int cin_cta = a.Cin / S;                      // input channels of this CTA (multiple of 16)
    float* sW = reinterpret_cast<float*>(smem);         // [NST][CK][K][NB]
    float* sX = sW + NST * CK * K * NB;                 // [TTP][cin_cta]
    float* sP = sX + TTP * cin_cta;                     // [TT][NB] partial tile (split-K only)
    uint64_t* bars = reinterpret_cast<uint64_t*>(sP + TT * NB);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = blockIdx.x;                        // cluster rank == K slice
    const int mtiles = (a.T + TT - 1) / TT;
    const int mt = blockIdx.y % mtiles, nb = blockIdx.y / mtiles, b = blockIdx.z;
    const int t0 = mt * TT, ci0 = rank * cin_cta;
    const int nch = cin_cta / CK;
    const uint32_t bar0 = smem_u32(bars);
    const uint32_t stage_bytes = (uint32_t)(CK * K * NB * 4);
    const float* wbase = a.w + ((size_t)ci0 * K) * a.Cout_w + (size_t)nb * NB;
    auto issue = [&](int c) {  // warp 0: one bulk copy per (ci, tap) row of 192 columns (768 B), or one per stage when rows are contiguous
        const int st = c % NST;
        if (lane == 0) mbar_expect_tx(bar0 + 8u * st, stage_bytes);
        __syncwarp();
        const float* src = wbase + (size_t)c * CK * K * a.Cout_w;
        if (a.Cout_w == NB) {
            if (lane == 0) bulk_g2s(smem_u32(sW + (size_t)st * CK * K * NB), src, stage_bytes, bar0 + 8u * st);
        } else {
            for (int r = lane; r < CK * K; r += 32) bulk_g2s(smem_u32(sW + ((size_t)st * CK * K + r) * NB), src + (size_t)r * a.Cout_w, NB * 4, bar0 + 8u * st);
        }
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; i++) mbar_init(bar0 + 8u * i, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (warp == 0)
        for (int c = 0; c < NST && c < nch; c++) issue(c);  // weights do not depend on the upstream kernel
    pdl_wait();
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int len = a.lens ? a.lens[b] : a.T;
    // ---- stage the input tile [TTP][cin_cta] (zero padding, x * x_mask)
    if (a.plain_C) {
        for (int i = threadIdx.x; i < cin_cta * TTP; i += 128) {
            const int ci = i / TTP, p = i - ci * TTP, t = t0 - PAD + p, cg_ = ci0 + ci;  // time fastest: each row segment is contiguous in HBM
            const float* src = a.plain[cg_ / a.plain_C] + ((size_t)b * a.plain_C + cg_ % a.plain_C) * a.T;
            sX[p * cin_cta + ci] = (t >= 0 && t < a.T && (!a.in_mask || t < len)) ? src[t] : 0.f;
        }
    } else {
        const float4* x4 = reinterpret_cast<const float4*>(a.x) + ((size_t)b * (a.Cin_total / 4) + (a.cin_off + ci0) / 4) * a.T;
        const int ncg = cin_cta / 4;
        for (int i = threadIdx.x; i < ncg * TTP; i += 128) {
            const int p = i / ncg, cg = i - p * ncg, t = t0 - PAD + p;  // cg fastest: conflict-free 16-byte shared stores
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t >= 0 && t < a.T && (!a.in_mask || t < len)) v = x4[(size_t)cg * a.T + t];
            *reinterpret_cast<float4*>(&sX[p * cin_cta + cg * 4]) = v;
        }
    }
    __syncthreads();
    float acc[4][6];
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int e = 0; e < 6; e++) acc[k][e] = 0.f;
    for (int c = 0; c < nch; c++) {
        const int st = c % NST;
        mbar_wait(bar0 + 8u * st, (c / NST) & 1);
        const float* W = sW + (size_t)st * CK * K * NB;
#pragma unroll
        for (int c4 = 0; c4 < CK; c4 += 4) {
            // activations of 4 input channels at the K + 3 time positions this warp needs (warp-uniform 16-byte loads)
            float xv[K + 3][4];
#pragma unroll
            for (int p = 0; p < K + 3; p++) {
                const float4 v = *reinterpret_cast<const float4*>(&sX[(4 * warp + p) * cin_cta + c * CK + c4]);
                xv[p][0] = v.x; xv[p][1] = v.y; xv[p][2] = v.z; xv[p][3] = v.w;
            }
#pragma unroll
            for (int e = 0; e < 4; e++) {
#pragma unroll
                for (int j = 0; j < K; j++) {  // fixed (ci ascending, tap ascending) summation order
                    const float* wr = W + ((c4 + e) * K + j) * NB;
                    const float4 wA = *reinterpret_cast<const float4*>(wr + 4 * lane);
                    const float2 wB = *reinterpret_cast<const float2*>(wr + 128 + 2 * lane);
#pragma unroll
                    for (int k = 0; k < 4; k++) {
                        const float x = xv[k + j][e];
                        acc[k][0] = fmaf(x, wA.x, acc[k][0]); acc[k][1] = fmaf(x, wA.y, acc[k][1]); acc[k][2] = fmaf(x, wA.z, acc[k][2]);
                        acc[k][3] = fmaf(x, wA.w, acc[k][3]); acc[k][4] = fmaf(x, wB.x, acc[k][4]); acc[k][5] = fmaf(x, wB.y, acc[k][5]);
                    }
                }
            }
        }
        __syncthreads();  // every warp is done with stage st
        if (warp == 0 && c + NST < nch) issue(c + NST);
    }
    // ---- epilogue of one finished row (all 192 channels of this column block live in one warp: 6 per lane)
    const int co = a.cout_off + nb * NB;
    const int cA = co + 4 * lane, cB = co + 128 + 2 * lane;
    auto finish_row = [&](int t, float* v) {
        float4 bA = a.bias ? *reinterpret_cast<const float4*>(a.bias + cA - a.cout_off) : make_float4(0.f, 0.f, 0.f, 0.f);
        float2 bB = a.bias ? *reinterpret_cast<const float2*>(a.bias + cB - a.cout_off) : make_float2(0.f, 0.f);
        if (a.bias_b) {
            const float4 b2 = *reinterpret_cast<const float4*>(a.bias_b + (size_t)b * a.bias_b_stride + cA - a.cout_off);
            const float2 b3 = *reinterpret_cast<const float2*>(a.bias_b + (size_t)b * a.bias_b_stride + cB - a.cout_off);
            bA.x += b2.x; bA.y += b2.y; bA.z += b2.z; bA.w += b2.w; bB.x += b3.x; bB.y += b3.y;
        }
        v[0] += bA.x; v[1] += bA.y; v[2] += bA.z; v[3] += bA.w; v[4] += bB.x; v[5] += bB.y;
        if (a.relu) {
#pragma unroll
            for (int e = 0; e < 6; e++) v[e] = fmaxf(v[e], 0.f);
        }
        if (a.mask_pre && t >= len) {
#pragma unroll
            for (int e = 0; e < 6; e++) v[e] = 0.f;
        }
        float4* y4 = reinterpret_cast<float4*>(a.y) + (size_t)b * (a.Cout_total / 4) * a.T;
        if (a.gamma) {  // y = LN(res + v): statistics are warp-uniform, so every lane takes part even when t >= T
            float rr[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (t < a.T) {
                const float4* r4 = reinterpret_cast<const float4*>(a.res) + (size_t)b * (a.res_C_total / 4) * a.T;
                const float4 rA = r4[(size_t)lane * a.T + t];
                const float2 rB = *(reinterpret_cast<const float2*>(r4 + (size_t)(32 + (lane >> 1)) * a.T + t) + (lane & 1));
                rr[0] = rA.x; rr[1] = rA.y; rr[2] = rA.z; rr[3] = rA.w; rr[4] = rB.x; rr[5] = rB.y;
            }
            float s = 0.f;
#pragma unroll
            for (int e = 0; e < 6; e++) { v[e] += rr[e]; }
            s = ((v[0] + v[1]) + (v[2] + v[3])) + (v[4] + v[5]);
            s = warp_sum(s);
            const float mean = s / (float)NB;
            float q = 0.f;
#pragma unroll
            for (int e = 0; e < 6; e++) { const float d = v[e] - mean; q += d * d; }
            q = warp_sum(q);
            const float rstd = rsqrtf(q / (float)NB + 1e-5f);
            const float4 gA = *reinterpret_cast<const float4*>(a.gamma + 4 * lane), eA = *reinterpret_cast<const float4*>(a.beta + 4 * lane);
            const float2 gB = *reinterpret_cast<const float2*>(a.gamma + 128 + 2 * lane), eB = *reinterpret_cast<const float2*>(a.beta + 128 + 2 * lane);
            v[0] = (v[0] - mean) * rstd * gA.x + eA.x; v[1] = (v[1] - mean) * rstd * gA.y + eA.y; v[2] = (v[2] - mean) * rstd * gA.z + eA.z;
            v[3] = (v[3] - mean) * rstd * gA.w + eA.w; v[4] = (v[4] - mean) * rstd * gB.x + eB.x; v[5] = (v[5] - mean) * rstd * gB.y + eB.y;
        }
        if (t >= a.T) return;
        const float m = (a.out_mask && t >= len) ? 0.f : 1.f;
        y4[(size_t)(cA / 4) * a.T + t] = make_float4(v[0] * m, v[1] * m, v[2] * m, v[3] * m);
        *(reinterpret_cast<float2*>(y4 + (size_t)(cB / 4) * a.T + t) + ((cB >> 1) & 1)) = make_float2(v[4] * m, v[5] * m);
    };
    if (S == 1) {
#pragma unroll
        for (int k = 0; k < 4; k++) finish_row(t0 + 4 * warp + k, acc[k]);
        return;
    }
    // ---- split-K: partial tiles -> own shared memory -> cluster barrier -> each rank sums and finishes TT/S rows over DSMEM
#pragma unroll
    for (int k = 0; k < 4; k++) {
        float* pr = sP + (4 * warp + k) * NB;
        *reinterpret_cast<float4*>(pr + 4 * lane) = make_float4(acc[k][0], acc[k][1], acc[k][2], acc[k][3]);
        *reinterpret_cast<float2*>(pr + 128 + 2 * lane) = make_float2(acc[k][4], acc[k][5]);
    }
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
    const int rows = TT / S;
    for (int r = rank * rows + warp; r < (rank + 1) * rows; r += 4) {
        float v[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        const uint32_t local = smem_u32(sP + r * NB);
        for (int q = 0; q < S; q++) {  // fixed rank order
            uint32_t remote;
            asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(local), "r"(q));
            float4 pA; float2 pB;
            asm volatile("ld.shared::cluster.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(pA.x), "=f"(pA.y), "=f"(pA.z), "=f"(pA.w) : "r"(remote + 16u * lane));
            asm volatile("ld.shared::cluster.v2.f32 {%0,%1}, [%2];" : "=f"(pB.x), "=f"(pB.y) : "r"(remote + 512u + 8u * lane));
            v[0] += pA.x; v[1] += pA.y; v[2] += pA.z; v[3] += pA.w; v[4] += pB.x; v[5] += pB.y;
        }
        finish_row(t0 + r, v);
    }
    // no CTA may exit while a peer still reads its shared memory
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

inline size_t tok_gemm_smem(int K, int cin_cta) { return (size_t)3 * 16 * K * 192 * 4 + (size_t)(16 + K - 1) * cin_cta * 4 + 16 * 192 * 4 + 64; }

// Launch helper: picks the split so that ~128 CTAs exist; requires Cout (of this launch) % 192 == 0, Cin % (16 * split) == 0.
inline bool launch_tok_gemm(TokGemmArgs a, int K, int Cout, cudaStream_t st, int force_split = 0) {
    if (!(K == 1 || K == 3) || Cout % 192 || a.Cin % 16 || a.T < 1) return false;
    if (a.gamma && (Cout != 192 || a.cout_off != 0 || !a.res)) return false;
    if ((a.in_mask || a.out_mask || a.mask_pre) && !a.lens) return false;
    const int nbk = Cout / 192, mtiles = cdiv(a.T, 16);
    int S = 1;
    const long long base = (long long)nbk * mtiles * a.B;
    while (S < 8 && base * S < 120 && a.Cin % (16 * S * 2) == 0) S *= 2;
    if (force_split) S = force_split;
    if (a.Cin % (16 * S)) return false;
    a.ksplit = S;
    const size_t smem = tok_gemm_smem(K, a.Cin / S);
    if (smem > 227 * 1024) return false;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(S, nbk * mtiles, a.B); cfg.blockDim = dim3(128); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
    attr[1].id = cudaLaunchAttributeClusterDimension; attr[1].val.clusterDim.x = S; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 2;
    if (K == 1) BV2_CUDA(cudaLaunchKernelEx(&cfg, k_tok_gemm<1>, a)); else BV2_CUDA(cudaLaunchKernelEx(&cfg, k_tok_gemm<3>, a));
    return true;
}

inline void tok_init_device() {
    BV2_CUDA(cudaFuncSetAttribute(k_dds_layer<192>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dds_layer_smem(192)));
    BV2_CUDA(cudaFuncSetAttribute(k_tok_gemm<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    BV2_CUDA(cudaFuncSetAttribute(k_tok_gemm<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
}

}  // namespace bv2
