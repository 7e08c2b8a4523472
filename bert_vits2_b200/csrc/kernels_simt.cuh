// fp32 SIMT kernels of the VITS2 infer path, all on the c4 activation layout (common.cuh).
// These are (1) the exact-fp32 path for everything that feeds ceil(durations) (text encoder, SDP, DP:
// SURVEY.md §7 H1) and (2) the fallback/baseline for the stages whose dense contractions run on wgmma
// (tc_conv.cuh).  Each kernel cites the reference op sequence it replaces.
#pragma once
#include "common.cuh"

namespace bv2 {

// ------------------------------------------------------------------------------------------------
// layout conversion
// ------------------------------------------------------------------------------------------------
// plain [B][C][Tsrc] (row stride src_ld) -> c4 [B][Ctot/4][T][4] at channel offset c_off; optional x_mask.
__global__ void k_plain_to_c4(const float* __restrict__ src, int C, long long src_bstride, int src_ld,
                              float* __restrict__ dst, int Ctot, int c_off, int T, const int* __restrict__ lens,
                              float scale) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int cg = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    float m = (lens && t >= lens[b]) ? 0.f : scale;
    const float* s = src + (size_t)b * src_bstride + (size_t)(cg * 4) * src_ld + t;
    float4 v;
    v.x = s[0] * m;
    v.y = (cg * 4 + 1 < C) ? s[src_ld] * m : 0.f;
    v.z = (cg * 4 + 2 < C) ? s[2 * (size_t)src_ld] * m : 0.f;
    v.w = (cg * 4 + 3 < C) ? s[3 * (size_t)src_ld] * m : 0.f;
    reinterpret_cast<float4*>(dst)[((size_t)b * (Ctot / 4) + c_off / 4 + cg) * T + t] = v;
}

// c4 [B][Ctot/4][T][4] channels [c_off, c_off+C) -> plain [B][C][Tdst] (first Tdst<=T steps)
__global__ void k_c4_to_plain(const float* __restrict__ src, int Ctot, int c_off, int T, float* __restrict__ dst,
                              int C, int Tdst) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int cg = blockIdx.y, b = blockIdx.z;
    if (t >= Tdst) return;
    float4 v = reinterpret_cast<const float4*>(src)[((size_t)b * (Ctot / 4) + c_off / 4 + cg) * T + t];
    float* d = dst + ((size_t)b * C + cg * 4) * Tdst + t;
    d[0] = v.x;
    if (cg * 4 + 1 < C) d[Tdst] = v.y;
    if (cg * 4 + 2 < C) d[2 * (size_t)Tdst] = v.z;
    if (cg * 4 + 3 < C) d[3 * (size_t)Tdst] = v.w;
}

// ------------------------------------------------------------------------------------------------
// generic dense Conv1d (stride 1), c4 in / c4 out.  Replaces F.conv1d call sites
// (reference attentions.py:264-270,439-445; modules.py:193,203,301-305; models.py:286-297,378-399,539-554).
// ------------------------------------------------------------------------------------------------
struct ConvArgs {
    const float* x = nullptr;  // c4 [B][Cin_total/4][T][4]
    int Cin_total = 0, cin_off = 0, Cin = 0;
    const float* w = nullptr;  // packed [Cin][K][Cout_w] (co fastest)
    int Cout_w = 0;
    const float* bias = nullptr;    // [Cout] or null
    const float* bias_b = nullptr;  // per-batch bias (speaker conditioning), row b at bias_b + b*bias_b_stride
    int bias_b_stride = 0;
    float* y = nullptr;  // c4 [B][Cout_total/4][T][4]
    int Cout_total = 0, cout_off = 0, Cout = 0;
    int T = 0, B = 0;
    int t_begin = 0, t_end = -1;  // output rows [t_begin, t_end) are computed and stored (t_end = -1: all T); reads still see all T rows
    int K = 1, dil = 1, pad = 0;
    float in_slope = 1.f;  // leaky-relu on the input (1 = identity)
    int in_mask = 0;       // input *= (t < lens[b])
    int act = 0;           // 1 = relu
    int res_mode = 0;      // 1: v += res ; 2: v = res - v
    const float* res = nullptr;
    int res_C_total = 0, res_c_off = 0;
    int accumulate = 0;    // v += y_old
    float out_scale = 1.f;
    int out_mask = 0;      // v *= (t < lens[b])
    const int* lens = nullptr;
};

// Tile = (16*NI time steps) x (4*CGN output channels), 16*CGN threads, each thread NI x 4 outputs.
// <8,16>: 128 x 64 tile for long sequences; <1,4>: 16 x 16 tile so that token-rate tensors (T ~ 256) still spread over
// >= 100 CTAs (the text encoder / duration predictors are latency-bound, SURVEY.md §7 H3).
// KS > 1: intra-CTA split of the input-channel reduction (KS thread groups each take CIT/KS channels of every chunk and
// the partial sums are combined through shared memory): the token-rate convs run at ~1 CTA per SM, so instruction
// latency, not throughput, bounds them.
template <int K, int NI, int CGN, int CIT, int KS = 1>
__global__ void __launch_bounds__(16 * CGN * KS) k_conv1d_c4(ConvArgs a) {
    pdl_wait();
    constexpr int TT = 16 * NI, COT = 4 * CGN, MAXD = 5, NTHR = 16 * CGN * KS, NT1 = 16 * CGN;
    constexpr int XW = TT + (K - 1) * MAXD;
    static_assert(KS == 1 || NI == 1, "split reduction only for the small tile");
    __shared__ float sx[CIT][XW];
    __shared__ __align__(16) float sw[CIT][K][COT];
    __shared__ __align__(16) float sred[KS > 1 ? KS : 1][KS > 1 ? NT1 : 1][4];
    const int tid = threadIdx.x % NT1, ks = threadIdx.x / NT1, tl = tid & 15, cgo = tid >> 4;
    const int b = blockIdx.z, t0 = a.t_begin + blockIdx.x * TT, co0 = blockIdx.y * COT;
    const int len = a.lens ? a.lens[b] : a.T, t_end = a.t_end < 0 ? a.T : a.t_end;
    const int xw = TT + (K - 1) * a.dil;
    float acc[NI][4];
#pragma unroll
    for (int i = 0; i < NI; i++) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const float4* x4 = reinterpret_cast<const float4*>(a.x) + ((size_t)b * (a.Cin_total / 4) + a.cin_off / 4) * a.T;

    for (int c0 = 0; c0 < a.Cin; c0 += CIT) {
        for (int i = threadIdx.x; i < (CIT / 4) * xw; i += NTHR) {
            int g = i / xw, p = i - g * xw;
            int t = t0 - a.pad + p;
            int cg = c0 / 4 + g;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (cg * 4 < a.Cin && t >= 0 && t < a.T && (!a.in_mask || t < len)) {
                v = x4[(size_t)cg * a.T + t];
                if (a.in_slope != 1.f) {
                    v.x = lrelu(v.x, a.in_slope); v.y = lrelu(v.y, a.in_slope);
                    v.z = lrelu(v.z, a.in_slope); v.w = lrelu(v.w, a.in_slope);
                }
            }
            sx[g * 4 + 0][p] = v.x; sx[g * 4 + 1][p] = v.y; sx[g * 4 + 2][p] = v.z; sx[g * 4 + 3][p] = v.w;
        }
        for (int i = threadIdx.x; i < CIT * K * (COT / 4); i += NTHR) {
            int c4i = i % (COT / 4), r = i / (COT / 4);
            int j = r % K, ci = r / K;
            int co = co0 + c4i * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (c0 + ci < a.Cin && co < a.Cout)
                v = *reinterpret_cast<const float4*>(a.w + ((size_t)(c0 + ci) * K + j) * a.Cout_w + co);
            *reinterpret_cast<float4*>(&sw[ci][j][c4i * 4]) = v;
        }
        __syncthreads();
#pragma unroll 2
        for (int ci = ks * (CIT / KS); ci < (ks + 1) * (CIT / KS); ci++) {
#pragma unroll
            for (int j = 0; j < K; j++) {
                const float4 w4 = *reinterpret_cast<const float4*>(&sw[ci][j][cgo * 4]);
                const float* xr = &sx[ci][tl + j * a.dil];
#pragma unroll
                for (int i = 0; i < NI; i++) {
                    float xv = xr[16 * i];
                    acc[i][0] = fmaf(xv, w4.x, acc[i][0]);
                    acc[i][1] = fmaf(xv, w4.y, acc[i][1]);
                    acc[i][2] = fmaf(xv, w4.z, acc[i][2]);
                    acc[i][3] = fmaf(xv, w4.w, acc[i][3]);
                }
            }
        }
        __syncthreads();
    }
    if (KS > 1) {
        *reinterpret_cast<float4*>(sred[ks][tid]) = make_float4(acc[0][0], acc[0][1], acc[0][2], acc[0][3]);
        __syncthreads();
        if (ks != 0) return;
#pragma unroll
        for (int q = 1; q < KS; q++) {
            const float4 v = *reinterpret_cast<const float4*>(sred[q][tid]);
            acc[0][0] += v.x; acc[0][1] += v.y; acc[0][2] += v.z; acc[0][3] += v.w;
        }
    }
    const int co = co0 + cgo * 4;
    if (co >= a.Cout) return;
    float4 bz = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a.bias) bz = *reinterpret_cast<const float4*>(a.bias + co);
    if (a.bias_b) {
        float4 b2 = *reinterpret_cast<const float4*>(a.bias_b + (size_t)b * a.bias_b_stride + co);
        bz.x += b2.x; bz.y += b2.y; bz.z += b2.z; bz.w += b2.w;
    }
    float4* y4 = reinterpret_cast<float4*>(a.y) + ((size_t)b * (a.Cout_total / 4) + (a.cout_off + co) / 4) * a.T;
    const float4* r4 = a.res ? reinterpret_cast<const float4*>(a.res) +
                                   ((size_t)b * (a.res_C_total / 4) + (a.res_c_off + co) / 4) * a.T
                             : nullptr;
#pragma unroll
    for (int i = 0; i < NI; i++) {
        int t = t0 + tl + 16 * i;
        if (t >= t_end) continue;  // stores, residual and accumulate reads stay inside the window
        float4 v = make_float4(acc[i][0] + bz.x, acc[i][1] + bz.y, acc[i][2] + bz.z, acc[i][3] + bz.w);
        if (a.act == 1) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        if (a.res_mode) {
            float4 r = r4[t];
            if (a.res_mode == 1) { v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
            else { v.x = r.x - v.x; v.y = r.y - v.y; v.z = r.z - v.z; v.w = r.w - v.w; }
        }
        if (a.accumulate) { float4 o = y4[t]; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
        float s = a.out_scale;
        if (a.out_mask && t >= len) s = 0.f;
        v.x *= s; v.y *= s; v.z *= s; v.w *= s;
        y4[t] = v;
    }
}

// The tile shape (and with it the split of the channel reduction) is chosen for the whole length a.T, so a windowed launch keeps the
// reduction order of every output; only the tiles covering the window are launched.
template <int K>
inline void launch_conv1d_k(const ConvArgs& a, cudaStream_t st) {
    const long long big_ctas = (long long)cdiv(a.T, 128) * cdiv(a.Cout, 64) * a.B;
    const int rows = (a.t_end < 0 ? a.T : a.t_end) - a.t_begin;
    if (big_ctas >= 96) {
        dim3 grid(cdiv(rows, 128), cdiv(a.Cout, 64), a.B);
        launch_pdl(k_conv1d_c4<K, 8, 16, 8>, grid, dim3(256), 0, st, a);
    } else {
        dim3 grid(cdiv(rows, 16), cdiv(a.Cout, 16), a.B);
        launch_pdl(k_conv1d_c4<K, 1, 4, 32, 4>, grid, dim3(256), 0, st, a);
    }
}

inline void launch_conv1d(const ConvArgs& a, cudaStream_t st) {
    BV2_CHECK(a.dil <= 5 && a.Cin % 4 == 0 && a.Cout % 4 == 0 && a.cin_off % 4 == 0 && a.cout_off % 4 == 0, "conv1d shape");
    BV2_CHECK(0 <= a.t_begin && a.t_begin < (a.t_end < 0 ? a.T : a.t_end) && a.t_end <= a.T, "conv1d output window");
    switch (a.K) {
        case 1: launch_conv1d_k<1>(a, st); break;
        case 3: launch_conv1d_k<3>(a, st); break;
        case 5: launch_conv1d_k<5>(a, st); break;
        case 7: launch_conv1d_k<7>(a, st); break;
        case 11: launch_conv1d_k<11>(a, st); break;
        default: throw Error(-2, "conv1d: unsupported kernel size " + std::to_string(a.K));
    }
    BV2_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------------
// ConvTranspose1d (Generator ups, reference models.py:543-545), K % u == 0, padding (K-u)/2, c4 in/out.
// out[n] = bias + sum_{ci} sum_{m} x[ci][(n+p)/u - m] * w[ci][(n+p)%u + m*u][co]
// ------------------------------------------------------------------------------------------------
struct ConvTArgs {
    const float* x; int Cin, Tin;
    const float* w;  // packed [Cin][K][Cout]
    const float* bias;
    float* y; int Cout, Tout;
    int K, u, p, B;
    float in_slope;
    int n_begin = 0, n_end = -1;  // output samples [n_begin, n_end) are computed and stored (n_end = -1: all Tout)
};

__global__ void __launch_bounds__(256) k_convT_c4(ConvTArgs a) {
    constexpr int TT = 128, COT = 64, CIT = 8, XW = 80, KMAX = 16;
    __shared__ float sx[CIT][XW];
    __shared__ __align__(16) float sw[CIT][KMAX][COT];
    const int tid = threadIdx.x, tl = tid & 15, cgo = tid >> 4;
    const int b = blockIdx.z, n0 = a.n_begin + blockIdx.x * TT, co0 = blockIdx.y * COT;
    const int n_end = a.n_end < 0 ? a.Tout : a.n_end;
    const int taps = a.K / a.u;
    const int i_base = (n0 + a.p) / a.u - (taps - 1);
    const int xw = (TT - 1 + a.p + n0) / a.u - i_base + 1;  // <= TT/u + taps
    int ih[8], rr[8];
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int q = n0 + tl + 16 * i + a.p;
        ih[i] = q / a.u - i_base;
        rr[i] = q % a.u;
    }
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; i++) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    const float4* x4 = reinterpret_cast<const float4*>(a.x) + (size_t)b * (a.Cin / 4) * a.Tin;
    for (int c0 = 0; c0 < a.Cin; c0 += CIT) {
        for (int i = tid; i < 2 * xw; i += 256) {
            int g = i >= xw ? 1 : 0, p = i - g * xw;
            int t = i_base + p;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (t >= 0 && t < a.Tin) {
                v = x4[(size_t)(c0 / 4 + g) * a.Tin + t];
                v.x = lrelu(v.x, a.in_slope); v.y = lrelu(v.y, a.in_slope);
                v.z = lrelu(v.z, a.in_slope); v.w = lrelu(v.w, a.in_slope);
            }
            sx[g * 4 + 0][p] = v.x; sx[g * 4 + 1][p] = v.y; sx[g * 4 + 2][p] = v.z; sx[g * 4 + 3][p] = v.w;
        }
        for (int i = tid; i < CIT * a.K * (COT / 4); i += 256) {
            int c4i = i % (COT / 4), r = i / (COT / 4);
            int j = r % a.K, ci = r / a.K;
            int co = co0 + c4i * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (co < a.Cout) v = *reinterpret_cast<const float4*>(a.w + ((size_t)(c0 + ci) * a.K + j) * a.Cout + co);
            *reinterpret_cast<float4*>(&sw[ci][j][c4i * 4]) = v;
        }
        __syncthreads();
        for (int ci = 0; ci < CIT; ci++) {
            for (int m = 0; m < taps; m++) {
#pragma unroll
                for (int i = 0; i < 8; i++) {
                    float xv = sx[ci][ih[i] - m];
                    const float4 w4 = *reinterpret_cast<const float4*>(&sw[ci][rr[i] + m * a.u][cgo * 4]);
                    acc[i][0] = fmaf(xv, w4.x, acc[i][0]);
                    acc[i][1] = fmaf(xv, w4.y, acc[i][1]);
                    acc[i][2] = fmaf(xv, w4.z, acc[i][2]);
                    acc[i][3] = fmaf(xv, w4.w, acc[i][3]);
                }
            }
        }
        __syncthreads();
    }
    const int co = co0 + cgo * 4;
    if (co >= a.Cout) return;
    float4 bz = *reinterpret_cast<const float4*>(a.bias + co);
    float4* y4 = reinterpret_cast<float4*>(a.y) + ((size_t)b * (a.Cout / 4) + co / 4) * a.Tout;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int n = n0 + tl + 16 * i;
        if (n < n_end) y4[n] = make_float4(acc[i][0] + bz.x, acc[i][1] + bz.y, acc[i][2] + bz.z, acc[i][3] + bz.w);
    }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm over channels per time step (reference modules.py:26-29 / attentions.py:21-24), optional
// residual input (Encoder: norm(x + y), attentions.py:114,118), optional exact-erf GELU (DDSConv,
// modules.py:123-127) and second residual after the activation (DDSConv x = x + y, :129).
// 8 lanes cooperate on one time step; warp-shuffle reductions.
// ------------------------------------------------------------------------------------------------
struct LnArgs {
    const float* x; const float* add;  // y_in = x + add (add may be null)
    const float* gamma; const float* beta;
    float* y;
    const float* post_res;  // y = post_res + f(LN(..)) if non-null
    int C, T, B;
    int gelu;       // apply exact GELU after LN
    int relu_in;    // apply relu to input before LN (DurationPredictor: relu then norm, models.py:291-292)
    int out_mask; const int* lens;
    float eps;
    // optional fused depthwise k=3 dilated conv in front of the norm (DDSConv: norms_1(convs_sep(x * x_mask)), modules.py:122-123)
    const float* dw_w = nullptr; const float* dw_b = nullptr; int dw_dil = 1;
};

__global__ void __launch_bounds__(256) k_layernorm_c4(LnArgs a) {
    pdl_wait();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int part = lane & 7, tsub = lane >> 3;
    const int t = (blockIdx.x * 8 + warp) * 4 + tsub;
    const int b = blockIdx.y;
    const int ncg = a.C / 4;
    const bool valid = t < a.T;
    const float4* x4 = reinterpret_cast<const float4*>(a.x) + (size_t)b * ncg * a.T;
    const float4* a4 = a.add ? reinterpret_cast<const float4*>(a.add) + (size_t)b * ncg * a.T : nullptr;
    float4 v[8];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int cg = part + 8 * i;
        v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (valid && cg < ncg && a.dw_w) {
            const int len = a.lens[b];
            float4 acc = *reinterpret_cast<const float4*>(a.dw_b + cg * 4);
            const float* wc = a.dw_w + cg * 4 * 3;
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const int tt = t + (j - 1) * a.dw_dil;
                if (tt >= 0 && tt < a.T && tt < len) {
                    const float4 xv = x4[(size_t)cg * a.T + tt];
                    acc.x = fmaf(xv.x, wc[0 * 3 + j], acc.x); acc.y = fmaf(xv.y, wc[1 * 3 + j], acc.y);
                    acc.z = fmaf(xv.z, wc[2 * 3 + j], acc.z); acc.w = fmaf(xv.w, wc[3 * 3 + j], acc.w);
                }
            }
            v[i] = acc;
            s += (acc.x + acc.y) + (acc.z + acc.w);
        } else if (valid && cg < ncg) {
            v[i] = x4[(size_t)cg * a.T + t];
            if (a4) { float4 r = a4[(size_t)cg * a.T + t]; v[i].x += r.x; v[i].y += r.y; v[i].z += r.z; v[i].w += r.w; }
            if (a.relu_in) { v[i].x = fmaxf(v[i].x, 0.f); v[i].y = fmaxf(v[i].y, 0.f); v[i].z = fmaxf(v[i].z, 0.f); v[i].w = fmaxf(v[i].w, 0.f); }
            s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
        }
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    const float mean = s / (float)a.C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int cg = part + 8 * i;
        if (cg < ncg) {
            float dx = v[i].x - mean, dy = v[i].y - mean, dz = v[i].z - mean, dw = v[i].w - mean;
            q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
        }
    }
    q += __shfl_xor_sync(0xffffffffu, q, 1);
    q += __shfl_xor_sync(0xffffffffu, q, 2);
    q += __shfl_xor_sync(0xffffffffu, q, 4);
    const float rstd = rsqrtf(q / (float)a.C + a.eps);
    if (!valid) return;
    float m = 1.f;
    if (a.out_mask && t >= a.lens[b]) m = 0.f;
    float4* y4 = reinterpret_cast<float4*>(a.y) + (size_t)b * ncg * a.T;
    const float4* p4 = a.post_res ? reinterpret_cast<const float4*>(a.post_res) + (size_t)b * ncg * a.T : nullptr;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        int cg = part + 8 * i;
        if (cg >= ncg) continue;
        float4 g = *reinterpret_cast<const float4*>(a.gamma + cg * 4);
        float4 be = *reinterpret_cast<const float4*>(a.beta + cg * 4);
        float4 o;
        o.x = (v[i].x - mean) * rstd * g.x + be.x;
        o.y = (v[i].y - mean) * rstd * g.y + be.y;
        o.z = (v[i].z - mean) * rstd * g.z + be.z;
        o.w = (v[i].w - mean) * rstd * g.w + be.w;
        if (a.gelu) { o.x = gelu_erf(o.x); o.y = gelu_erf(o.y); o.z = gelu_erf(o.z); o.w = gelu_erf(o.w); }
        if (p4) { float4 r = p4[(size_t)cg * a.T + t]; o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w; }
        o.x *= m; o.y *= m; o.z *= m; o.w *= m;
        y4[(size_t)cg * a.T + t] = o;
    }
}

inline void launch_layernorm(const LnArgs& a, cudaStream_t st) {
    BV2_CHECK(a.C % 4 == 0 && a.C <= 256, "layernorm C");
    dim3 grid(cdiv(a.T, 32), a.B);
    launch_pdl(k_layernorm_c4, grid, dim3(256), 0, st, a);
}

// ------------------------------------------------------------------------------------------------
// y[b][co] = bias[co] + sum_ci W[co][ci] * g[b][ci]   -- every speaker-conditioning projection of the
// model in ONE launch (dec.cond, sdp.cond, dp.cond, Encoder.spk_emb_linear x5, WN.cond_layer x4).
// One warp per output element.
// ------------------------------------------------------------------------------------------------
__global__ void k_linear_g(const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ g,
                           float* __restrict__ y, int Cout, int Cin) {
    int co = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    int b = blockIdx.y, lane = threadIdx.x & 31;
    if (co >= Cout) return;
    const float* w = W + (size_t)co * Cin;
    const float* gv = g + (size_t)b * Cin;
    float s = 0.f;
    for (int i = lane; i < Cin; i += 32) s = fmaf(w[i], gv[i], s);
    s = warp_sum(s);
    if (lane == 0) y[(size_t)b * Cout + co] = s + bias[co];
}

__global__ void k_gather_rows(const float* __restrict__ table, const long long* __restrict__ idx, float* __restrict__ out, int C, int nrows) {
    int b = blockIdx.x;
    const long long r = min(max(idx[b], 0ll), (long long)nrows - 1);  // out-of-range ids are reported by k_validate_inputs; never read out of bounds
    for (int i = threadIdx.x; i < C; i += blockDim.x) out[(size_t)b * C + i] = table[(size_t)r * C + i];
}

// Speaker mix (bv2_infer_begin_mix): out[b][c] = sum_k w[b][k] * table[id[b][k]][c], summed in k order with one fp32 rounding per
// product and per sum (__fmul_rn / __fadd_rn: no FMA contraction, so np.float32 in the same order gives the same bits).  One block
// per b.  Validates the mix like k_validate_inputs: ORs 8 into *err for an id outside [0, nrows) (the read is clamped) and 32 for
// a non-finite weight.
__global__ void k_speaker_mix(const float* __restrict__ table, const long long* __restrict__ ids, const float* __restrict__ w, int K,
                              float* __restrict__ out, int C, int nrows, int* __restrict__ err) {
    const int b = blockIdx.x;
    const long long* id = ids + (size_t)b * K;
    const float* wb = w + (size_t)b * K;
    int bad = 0;
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
        float acc = 0.f;
        for (int k = 0; k < K; k++) {
            const long long r = id[k];
            const float wk = wb[k];
            if (r < 0 || r >= nrows) bad |= 8;
            if (!isfinite(wk)) bad |= 32;
            const float p = __fmul_rn(wk, table[(size_t)min(max(r, 0ll), (long long)nrows - 1) * C + i]);
            acc = k ? __fadd_rn(acc, p) : p;
        }
        out[(size_t)b * C + i] = acc;
    }
    if (bad && threadIdx.x == 0) atomicOr(err, bad);  // thread 0 walks every k for channel 0
}

// Input validation (the reference raises IndexError from nn.Embedding / a shape error for bad lengths; reference
// models.py:378-384, 1046): ids must lie inside their tables and 1 <= x_lengths[b] <= T.  Writes a bit mask into *err
// (read back together with y_lengths: no extra synchronisation): 1 = phoneme id, 2 = tone, 4 = language, 8 = speaker id,
// 16 = x_lengths (32 = a non-finite speaker-mix weight, from k_speaker_mix).  Gather kernels clamp, so a bad id can never become
// an out-of-bounds access.
__global__ void k_validate_inputs(const long long* __restrict__ x, const long long* __restrict__ tone, const long long* __restrict__ lang,
                                  const long long* __restrict__ sid, const long long* __restrict__ lens, int B, int T, int n_vocab,
                                  int n_tones, int n_langs, int n_spk, int* __restrict__ err) {
    int bad = 0;
    const int n = B * T;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int b = i / T, t = i - b * T;
        const long long l = lens ? lens[b] : T;
        if (t >= l) continue;  // padding positions are never read as ids with an effect (masked)
        if (x && (x[i] < 0 || x[i] >= n_vocab)) bad |= 1;
        if (tone && (tone[i] < 0 || tone[i] >= n_tones)) bad |= 2;
        if (lang && (lang[i] < 0 || lang[i] >= n_langs)) bad |= 4;
    }
    if (blockIdx.x == 0)
        for (int b = threadIdx.x; b < B; b += blockDim.x) {
            if (sid && (sid[b] < 0 || sid[b] >= n_spk)) bad |= 8;
            if (lens && (lens[b] < 1 || lens[b] > T)) bad |= 16;
        }
    if (bad) atomicOr(err, bad);
}

// ------------------------------------------------------------------------------------------------
// TextEncoder front end (reference models.py:378-394): h = (emb[x]+tone_emb[tone]+lang_emb[lang]+bert projections)
// * sqrt(H) * x_mask.  The three 1024->192 projections were accumulated into `proj` by one K=3072 conv.
// ------------------------------------------------------------------------------------------------
__global__ void k_embed_sum(const float* __restrict__ proj, const long long* __restrict__ x, const long long* __restrict__ tone,
                            const long long* __restrict__ lang, const float* __restrict__ emb, const float* __restrict__ temb,
                            const float* __restrict__ lemb, float* __restrict__ out, int H, int T, const int* __restrict__ lens,
                            float scale, int n_vocab, int n_tones, int n_langs) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int cg = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    size_t idx = ((size_t)b * (H / 4) + cg) * T + t;
    float4 p = reinterpret_cast<const float4*>(proj)[idx];
    long long xi = x[(size_t)b * T + t], ti = tone[(size_t)b * T + t], li = lang[(size_t)b * T + t];
    xi = min(max(xi, 0ll), (long long)n_vocab - 1); ti = min(max(ti, 0ll), (long long)n_tones - 1); li = min(max(li, 0ll), (long long)n_langs - 1);
    float4 e = *reinterpret_cast<const float4*>(emb + xi * H + cg * 4);
    float4 te = *reinterpret_cast<const float4*>(temb + ti * H + cg * 4);
    float4 le = *reinterpret_cast<const float4*>(lemb + li * H + cg * 4);
    float m = t < lens[b] ? scale : 0.f;
    float4 o;
    o.x = (((e.x + te.x) + le.x) + p.x) * m;
    o.y = (((e.y + te.y) + le.y) + p.y) * m;
    o.z = (((e.z + te.z) + le.z) + p.z) * m;
    o.w = (((e.w + te.w) + le.w) + p.w) * m;
    reinterpret_cast<float4*>(out)[idx] = o;
}

// x[b][c][t] = (x + add[b][c]) * mask   (Encoder speaker injection, reference attentions.py:107-111)
__global__ void k_add_bvec_mask(float* __restrict__ x, const float* __restrict__ add, int add_stride, int C, int T,
                                const int* __restrict__ lens) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int cg = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    size_t idx = ((size_t)b * (C / 4) + cg) * T + t;
    float4 v = reinterpret_cast<float4*>(x)[idx];
    float4 g = *reinterpret_cast<const float4*>(add + (size_t)b * add_stride + cg * 4);
    float m = t < lens[b] ? 1.f : 0.f;
    v.x = (v.x + g.x) * m; v.y = (v.y + g.y) * m; v.z = (v.z + g.z) * m; v.w = (v.w + g.w) * m;
    reinterpret_cast<float4*>(x)[idx] = v;
}

// ------------------------------------------------------------------------------------------------
// Windowed relative-position multi-head self-attention (reference attentions.py:272-322) in banded form:
//   scores[i,j] = q_i.k_j + [|j-i|<=w] q_i.Ek[j-i+w];  out_i = sum_j p_ij v_j + sum_r p_{i,i+r-w} Ev[r]
// (the reference's dense pad/reshape formulation, attentions.py:285-290,311-318,360-395, is 98.6 % zeros).
// qkv: c4 [B][3H/4][T][4] = (q already scaled by 1/sqrt(dk) via folded weights, k, v).  Online softmax over
// key chunks of 64; keys j >= len are excluded (== the reference's -1e4 fill, which underflows to 0).
// ------------------------------------------------------------------------------------------------
template <int DK>
__global__ void __launch_bounds__(128) k_attention_rel(const float* __restrict__ qkv, const float* __restrict__ rel_k,
                                                      const float* __restrict__ rel_v, float* __restrict__ out, int H, int T,
                                                      const int* __restrict__ lens, int window) {
    constexpr int QT = 16, KT = 64, NCG = DK / 4, VP = DK + 4, DPT = DK / 8;  // DPT dims per thread in PV phase
    static_assert(DK % 32 == 0, "DK");
    __shared__ __align__(16) float sq[QT][DK];
    __shared__ float srelq[QT][12];
    __shared__ float srelp[QT][12];
    __shared__ float sp[QT][KT];
    __shared__ __align__(16) float sv[KT][VP];
    const int tid = threadIdx.x;
    const int b = blockIdx.z, h = blockIdx.y, i0 = blockIdx.x * QT;
    const int len = lens ? lens[b] : T;
    const int nrel = 2 * window + 1;
    const int C3 = 3 * H;
    const float4* base = reinterpret_cast<const float4*>(qkv) + (size_t)b * (C3 / 4) * T;
    const float4* q4 = base + (size_t)(h * NCG) * T;
    const float4* k4 = base + (size_t)(H / 4 + h * NCG) * T;
    const float4* v4 = base + (size_t)(2 * H / 4 + h * NCG) * T;

    for (int i = tid; i < QT * NCG; i += 128) {
        int qi = i % QT, cg = i / QT;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i0 + qi < T) v = q4[(size_t)cg * T + i0 + qi];
        *reinterpret_cast<float4*>(&sq[qi][cg * 4]) = v;
    }
    for (int i = tid; i < QT * 12; i += 128) srelp[i / 12][i % 12] = 0.f;
    __syncthreads();
    for (int i = tid; i < QT * nrel; i += 128) {
        int qi = i / nrel, r = i % nrel;
        float s = 0.f;
        for (int d = 0; d < DK; d++) s = fmaf(sq[qi][d], rel_k[r * DK + d], s);
        srelq[qi][r] = s;
    }
    // softmax / PV roles
    const int row = tid >> 3, sub = tid & 7;
    float m_run = -INFINITY, l_run = 0.f;
    float acc[DPT];
#pragma unroll
    for (int d = 0; d < DPT; d++) acc[d] = 0.f;
    // score role
    const int kj = tid & 63, qh = tid >> 6;  // key within chunk, query half (8 queries each)
    __syncthreads();

    for (int j0 = 0; j0 < len; j0 += KT) {
        const int j = j0 + kj;
        // ---- scores
        {
            float kreg[DK];
            if (j < len) {
#pragma unroll
                for (int cg = 0; cg < NCG; cg++) {
                    float4 v = k4[(size_t)cg * T + j];
                    kreg[cg * 4] = v.x; kreg[cg * 4 + 1] = v.y; kreg[cg * 4 + 2] = v.z; kreg[cg * 4 + 3] = v.w;
                }
            } else {
#pragma unroll
                for (int d = 0; d < DK; d++) kreg[d] = 0.f;
            }
#pragma unroll
            for (int qq = 0; qq < 8; qq++) {
                const int qi = qh * 8 + qq;
                float s = 0.f;
#pragma unroll
                for (int cg = 0; cg < NCG; cg++) {
                    float4 qv = *reinterpret_cast<const float4*>(&sq[qi][cg * 4]);
                    s = fmaf(qv.x, kreg[cg * 4], s); s = fmaf(qv.y, kreg[cg * 4 + 1], s);
                    s = fmaf(qv.z, kreg[cg * 4 + 2], s); s = fmaf(qv.w, kreg[cg * 4 + 3], s);
                }
                int rel = j - (i0 + qi) + window;
                if (rel >= 0 && rel < nrel) s += srelq[qi][rel];
                sp[qi][kj] = (j < len) ? s : -INFINITY;
            }
        }
        // ---- V chunk to smem
        for (int i = tid; i < KT * NCG; i += 128) {
            int jj = i % KT, cg = i / KT;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (j0 + jj < len) v = v4[(size_t)cg * T + j0 + jj];
            *reinterpret_cast<float4*>(&sv[jj][cg * 4]) = v;
        }
        __syncthreads();
        // ---- online softmax: 8 threads per row, 8 keys each
        float mx = -INFINITY;
#pragma unroll
        for (int e = 0; e < 8; e++) mx = fmaxf(mx, sp[row][sub * 8 + e]);
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 4));
        const float m_new = fmaxf(m_run, mx);  // finite: chunk has >= 1 valid key
        const float scale = (m_run == -INFINITY) ? 0.f : expf(m_run - m_new);
        float ls = 0.f;
#pragma unroll
        for (int e = 0; e < 8; e++) {
            float p = expf(sp[row][sub * 8 + e] - m_new);  // exp(-inf) = 0 for excluded keys
            sp[row][sub * 8 + e] = p;
            ls += p;
        }
        ls += __shfl_xor_sync(0xffffffffu, ls, 1);
        ls += __shfl_xor_sync(0xffffffffu, ls, 2);
        ls += __shfl_xor_sync(0xffffffffu, ls, 4);
        l_run = l_run * scale + ls;
        m_run = m_new;
#pragma unroll
        for (int d = 0; d < DPT; d++) acc[d] *= scale;
        if (sub < nrel) srelp[row][sub] *= scale;
        if (sub + 8 < nrel) srelp[row][sub + 8] *= scale;
        __syncthreads();
        // ---- relative-value weights: p[i, i+r-w]
#pragma unroll
        for (int e = 0; e < 8; e++) {
            int jj = j0 + sub * 8 + e;
            int rel = jj - (i0 + row) + window;
            if (rel >= 0 && rel < nrel && jj < len) srelp[row][rel] += sp[row][sub * 8 + e];
        }
        // ---- PV
        const int kmax = min(KT, len - j0);
        for (int jj = 0; jj < kmax; jj++) {
            const float p = sp[row][jj];
#pragma unroll
            for (int d4 = 0; d4 < DPT / 4; d4++) {
                float4 v = *reinterpret_cast<const float4*>(&sv[jj][sub * DPT + d4 * 4]);
                acc[d4 * 4 + 0] = fmaf(p, v.x, acc[d4 * 4 + 0]);
                acc[d4 * 4 + 1] = fmaf(p, v.y, acc[d4 * 4 + 1]);
                acc[d4 * 4 + 2] = fmaf(p, v.z, acc[d4 * 4 + 2]);
                acc[d4 * 4 + 3] = fmaf(p, v.w, acc[d4 * 4 + 3]);
            }
        }
        __syncthreads();
    }
    // ---- finalize
    const int qi = i0 + row;
    if (qi >= T) return;
    float4* o4 = reinterpret_cast<float4*>(out) + ((size_t)b * (H / 4) + h * NCG) * T;
    const bool qvalid = qi < len && l_run > 0.f;
    const float inv = qvalid ? 1.f / l_run : 0.f;
#pragma unroll
    for (int d4 = 0; d4 < DPT / 4; d4++) {
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            int d = sub * DPT + d4 * 4 + e;
            float s = acc[d4 * 4 + e];
            for (int r = 0; r < nrel; r++) s = fmaf(srelp[row][r], rel_v[r * DK + d], s);
            o[e] = s * inv;
        }
        o4[(size_t)((sub * DPT) / 4 + d4) * T + qi] = make_float4(o[0], o[1], o[2], o[3]);
    }
}

// ConvFlow.pre (Conv1d 1->C, k=1) fused with DDSConv's "x = x + g" (reference modules.py:488, 119-120):
// out[b][c][t] = w[c]*z[b][ch][t] + bias[c] + cond[b][c][t]
__global__ void k_flow_pre(const float* __restrict__ z, int zch, const float* __restrict__ w, const float* __restrict__ bias,
                           const float* __restrict__ cond, float* __restrict__ out, int C, int T) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int cg = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    float x0 = z[((size_t)b * 2 + zch) * T + t];
    size_t idx = ((size_t)b * (C / 4) + cg) * T + t;
    float4 c = reinterpret_cast<const float4*>(cond)[idx];
    float4 wv = *reinterpret_cast<const float4*>(w + cg * 4);
    float4 bv = *reinterpret_cast<const float4*>(bias + cg * 4);
    float4 o = make_float4(fmaf(wv.x, x0, bv.x) + c.x, fmaf(wv.y, x0, bv.y) + c.y, fmaf(wv.z, x0, bv.z) + c.z,
                           fmaf(wv.w, x0, bv.w) + c.w);
    reinterpret_cast<float4*>(out)[idx] = o;
}

// ------------------------------------------------------------------------------------------------
// Inverse piecewise rational-quadratic spline with linear tails (reference transforms.py:49-96, 99-173),
// one thread per (b, t); h holds the 3*NB-1 ConvFlow.proj outputs in c4 (Cout padded to 32).
// Updates z[b][x1ch][t] in place, then masks both channels (modules.py:512).
// ------------------------------------------------------------------------------------------------
template <int NB>
__global__ void k_spline_inverse(const float* __restrict__ h, int HC, float* __restrict__ z, int x1ch, int T,
                                 const int* __restrict__ lens, float inv_sqrt_filter, float tail, float dconst) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int b = blockIdx.y;
    if (t >= T) return;
    const float mask = t < lens[b] ? 1.f : 0.f;
    float p[3 * NB];  // 3*NB-1 used
    const float4* h4 = reinterpret_cast<const float4*>(h) + (size_t)b * (HC / 4) * T;
#pragma unroll
    for (int cg = 0; cg < (3 * NB + 3) / 4; cg++) {
        float4 v = h4[(size_t)cg * T + t];
        if (cg * 4 + 0 < 3 * NB) p[cg * 4 + 0] = v.x * mask;
        if (cg * 4 + 1 < 3 * NB) p[cg * 4 + 1] = v.y * mask;
        if (cg * 4 + 2 < 3 * NB) p[cg * 4 + 2] = v.z * mask;
        if (cg * 4 + 3 < 3 * NB) p[cg * 4 + 3] = v.w * mask;
    }
    float* zb = z + (size_t)b * 2 * T;
    const float x = zb[(size_t)x1ch * T + t];
    const float x0 = zb[(size_t)(1 - x1ch) * T + t];
    float outv = x;
    if (x >= -tail && x <= tail) {
        const float min_bw = 1e-3f, min_bh = 1e-3f, min_d = 1e-3f;
        float cw[NB + 1], chh[NB + 1];
        // widths
        {
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < NB; i++) { p[i] *= inv_sqrt_filter; mx = fmaxf(mx, p[i]); }
            float s = 0.f, e[NB];
#pragma unroll
            for (int i = 0; i < NB; i++) { e[i] = expf(p[i] - mx); s += e[i]; }
            float c = 0.f;
            cw[0] = -tail;
#pragma unroll
            for (int i = 0; i < NB; i++) {
                float wdt = __fadd_rn(min_bw, __fmul_rn(1.f - min_bw * NB, e[i] / s));
                c += wdt;
                cw[i + 1] = __fadd_rn(__fmul_rn(2.f * tail, c), -tail);
            }
            cw[NB] = tail;
        }
        {
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < NB; i++) { p[NB + i] *= inv_sqrt_filter; mx = fmaxf(mx, p[NB + i]); }
            float s = 0.f, e[NB];
#pragma unroll
            for (int i = 0; i < NB; i++) { e[i] = expf(p[NB + i] - mx); s += e[i]; }
            float c = 0.f;
            chh[0] = -tail;
#pragma unroll
            for (int i = 0; i < NB; i++) {
                float hgt = __fadd_rn(min_bh, __fmul_rn(1.f - min_bh * NB, e[i] / s));
                c += hgt;
                chh[i + 1] = __fadd_rn(__fmul_rn(2.f * tail, c), -tail);
            }
            chh[NB] = tail;
        }
        // bin search on cumheights (last knot + 1e-6, transforms.py:44-46)
        int bin = -1;
#pragma unroll
        for (int i = 0; i <= NB; i++) {
            float loc = (i == NB) ? chh[NB] + 1e-6f : chh[i];
            bin += (x >= loc) ? 1 : 0;
        }
        bin = min(max(bin, 0), NB - 1);
        float in_cw = 0.f, in_bw = 0.f, in_ch = 0.f, in_h = 0.f, ud0 = 0.f, ud1 = 0.f;
#pragma unroll
        for (int i = 0; i < NB; i++) {
            if (i == bin) {
                in_cw = cw[i]; in_bw = cw[i + 1] - cw[i];
                in_ch = chh[i]; in_h = chh[i + 1] - chh[i];
                ud0 = (i == 0) ? dconst : p[2 * NB + i - 1];
                ud1 = (i == NB - 1) ? dconst : p[2 * NB + i];
            }
        }
        const float in_delta = in_h / in_bw;
        const float d0 = min_d + softplusf_(ud0);
        const float d1 = min_d + softplusf_(ud1);
        const float dx = x - in_ch;
        const float sdd = (d0 + d1) - 2.f * in_delta;
        const float aa = __fadd_rn(__fmul_rn(dx, sdd), __fmul_rn(in_h, in_delta - d0));
        const float bb = __fadd_rn(__fmul_rn(in_h, d0), -__fmul_rn(dx, sdd));
        const float cc = __fmul_rn(-in_delta, dx);
        const float disc = __fadd_rn(__fmul_rn(bb, bb), -__fmul_rn(__fmul_rn(4.f, aa), cc));
        const float root = (2.f * cc) / (-bb - sqrtf(fmaxf(disc, 0.f)));
        outv = __fadd_rn(__fmul_rn(root, in_bw), in_cw);
    }
    zb[(size_t)x1ch * T + t] = outv * mask;
    zb[(size_t)(1 - x1ch) * T + t] = x0 * mask;
}

// ------------------------------------------------------------------------------------------------
// Durations (reference models.py:1052-1057 + ElementwiseAffine reverse modules.py:397-399).  One block per b.
// z: SDP latent [B][2][T] (channel `zch` is logw after the final Flip bookkeeping); dp: c4 [B][4/4][T][4] ch 0.
// sdp_ratio_b / length_scale_b (optional, [B]): item b's own setting instead of the scalar (bv2_infer_begin_items).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_durations(const float* __restrict__ z, int zch, float ea_m, float ea_logs,
                                                   const float* __restrict__ dp, float sdp_ratio, float length_scale,
                                                   const float* __restrict__ sdp_ratio_b, const float* __restrict__ length_scale_b,
                                                   const int* __restrict__ lens, int T, float* __restrict__ logw_sdp,
                                                   float* __restrict__ logw_dp, float* __restrict__ w_ceil,
                                                   int* __restrict__ cum, long long* __restrict__ y_len,
                                                   const float* __restrict__ w_ceil_override) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int len = lens[b];
    if (sdp_ratio_b) sdp_ratio = sdp_ratio_b[b];
    if (length_scale_b) length_scale = length_scale_b[b];
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (int t0 = 0; t0 < T; t0 += 1024) {
        int t = t0 + tid;
        int wi = 0;
        if (t < T) {
            float mask = t < len ? 1.f : 0.f;
            float zs = z[((size_t)b * 2 + zch) * T + t];
            float ls = __fmul_rn(__fmul_rn(zs - ea_m, expf(-ea_logs)), mask);
            float ld = reinterpret_cast<const float4*>(dp)[(size_t)b * T + t].x;  // already masked
            logw_sdp[(size_t)b * T + t] = ls;
            logw_dp[(size_t)b * T + t] = ld;
            float lw = __fadd_rn(__fmul_rn(ls, sdp_ratio), __fmul_rn(ld, 1.f - sdp_ratio));
            float w = __fmul_rn(__fmul_rn(expf(lw), mask), length_scale);
            float wc = w_ceil_override ? w_ceil_override[(size_t)b * T + t] : ceilf(w);
            w_ceil[(size_t)b * T + t] = wc;
            wi = (int)wc;
        }
        // block inclusive scan
        int v = wi;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int n = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += n;
        }
        if (lane == 31) s_warp[warp] = v;
        __syncthreads();
        if (warp == 0) {
            int wv = s_warp[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                int n = __shfl_up_sync(0xffffffffu, wv, o);
                if (lane >= o) wv += n;
            }
            s_warp[lane] = wv;
        }
        __syncthreads();
        int incl = v + (warp ? s_warp[warp - 1] : 0) + s_carry;
        if (t < T) cum[(size_t)b * T + t] = incl;
        __syncthreads();
        if (tid == 1023) s_carry = incl;
        __syncthreads();
    }
    if (tid == 0) {
        int total = cum[(size_t)b * T + T - 1];
        y_len[b] = total < 1 ? 1 : total;
    }
}

// ------------------------------------------------------------------------------------------------
// Length regulation + prior sampling (reference models.py:1058-1071, commons.py:126-140): a gather by
// binary search on the duration cumsum instead of the reference's dense one-hot matmul.
// stats: c4 [B][2I/4][T][4] (m = channels [0,I), logs = [I,2I)).  One thread per (b, f, cg).
// noise_scale_b (optional, [B]): item b samples with noise_scale * noise_scale_b[b], rounded once (bv2_infer_begin_items).
// ------------------------------------------------------------------------------------------------
__global__ void k_expand_prior(const float* __restrict__ stats, const int* __restrict__ cum, const long long* __restrict__ y_len,
                               const int* __restrict__ lens, const float* __restrict__ noise, long long noise_bstride,
                               int noise_ld, float noise_scale, const float* __restrict__ noise_scale_b, int I, int T, int F,
                               float* __restrict__ m_out, float* __restrict__ logs_out, float* __restrict__ zp_out,
                               float* __restrict__ zp_c4, float* __restrict__ y_mask) {
    int f = blockIdx.x * blockDim.x + threadIdx.x;
    int cg = blockIdx.y, b = blockIdx.z;
    if (f >= F) return;
    if (noise_scale_b) noise_scale = __fmul_rn(noise_scale, noise_scale_b[b]);
    const int yl = (int)y_len[b];
    const int* cb = cum + (size_t)b * T;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f), lg = m;
    const int len = lens[b];
    if (f < yl) {
        int lo = 0, hi = T - 1;  // first tk with cum[tk] > f
        while (lo < hi) {
            int mid = (lo + hi) >> 1;
            if (cb[mid] > f) hi = mid; else lo = mid + 1;
        }
        if (cb[lo] > f && lo < len) {
            const float4* s4 = reinterpret_cast<const float4*>(stats) + (size_t)b * (2 * I / 4) * T;
            m = s4[(size_t)cg * T + lo];
            lg = s4[(size_t)(I / 4 + cg) * T + lo];
        }
    }
    if (cg == 0 && y_mask) y_mask[(size_t)b * F + f] = f < yl ? 1.f : 0.f;
    float n[4], mv[4] = {m.x, m.y, m.z, m.w}, lv[4] = {lg.x, lg.y, lg.z, lg.w}, zp[4];
#pragma unroll
    for (int e = 0; e < 4; e++) {
        n[e] = noise[(size_t)b * noise_bstride + (size_t)(cg * 4 + e) * noise_ld + f];
        zp[e] = __fadd_rn(mv[e], __fmul_rn(__fmul_rn(n[e], expf(lv[e])), noise_scale));
        size_t o = ((size_t)b * I + cg * 4 + e) * F + f;
        m_out[o] = mv[e];
        logs_out[o] = lv[e];
        zp_out[o] = zp[e];
    }
    reinterpret_cast<float4*>(zp_c4)[((size_t)b * (I / 4) + cg) * F + f] = make_float4(zp[0], zp[1], zp[2], zp[3]);
}

// attn[b,0,f,t] one-hot path (reference commons.py:126-140), returned by infer() for API compatibility.
__global__ void k_attn_path(const int* __restrict__ cum, const long long* __restrict__ y_len, const int* __restrict__ lens,
                            float* __restrict__ attn, int T, int F) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int f = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const int* cb = cum + (size_t)b * T;
    int hi = cb[t], lo = t ? cb[t - 1] : 0;
    float v = (f >= lo && f < hi && f < (int)y_len[b] && t < lens[b]) ? 1.f : 0.f;
    attn[((size_t)b * F + f) * T + t] = v;
}

// ------------------------------------------------------------------------------------------------
// WN gate (reference commons.py:98-105 via modules.py:200): acts = tanh(a[:H] + g[:H]) * sigmoid(a[H:] + g[H:])
// ------------------------------------------------------------------------------------------------
__global__ void k_wn_gate(const float* __restrict__ xin, const float* __restrict__ g, int g_stride, float* __restrict__ acts,
                          int H, int T) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int cg = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    const float4* x4 = reinterpret_cast<const float4*>(xin) + (size_t)b * (2 * H / 4) * T;
    float4 a = x4[(size_t)cg * T + t], s = x4[(size_t)(H / 4 + cg) * T + t];
    float4 ga = *reinterpret_cast<const float4*>(g + (size_t)b * g_stride + cg * 4);
    float4 gs = *reinterpret_cast<const float4*>(g + (size_t)b * g_stride + H + cg * 4);
    float4 o;
    o.x = tanhf(a.x + ga.x) * sigmoidf_(s.x + gs.x);
    o.y = tanhf(a.y + ga.y) * sigmoidf_(s.y + gs.y);
    o.z = tanhf(a.z + ga.z) * sigmoidf_(s.z + gs.z);
    o.w = tanhf(a.w + ga.w) * sigmoidf_(s.w + gs.w);
    reinterpret_cast<float4*>(acts)[((size_t)b * (H / 4) + cg) * T + t] = o;
}

// Physical channel flip of a c4 tensor (only needed when n_flow_layer is odd; flips are otherwise folded
// into the coupling weights at load time).
__global__ void k_flip_c4(const float* __restrict__ x, float* __restrict__ y, int C, int T) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int cg = blockIdx.y, b = blockIdx.z;
    if (t >= T) return;
    float4 v = reinterpret_cast<const float4*>(x)[((size_t)b * (C / 4) + (C / 4 - 1 - cg)) * T + t];
    reinterpret_cast<float4*>(y)[((size_t)b * (C / 4) + cg) * T + t] = make_float4(v.w, v.z, v.y, v.x);
}

// ------------------------------------------------------------------------------------------------
// Generator tail (reference models.py:553-555): leaky_relu(0.01) -> conv_post(C->1, k7, no bias) -> tanh.
// ------------------------------------------------------------------------------------------------
template <int C, int K>
__global__ void __launch_bounds__(256) k_conv_post_tanh(const float* __restrict__ x, const float* __restrict__ w,
                                                       float* __restrict__ y, int T, float slope, int t_begin, int t_end) {
    __shared__ float sw[C * K];
    for (int i = threadIdx.x; i < C * K; i += blockDim.x) sw[i] = w[i];  // [C][K]
    __syncthreads();
    int t = t_begin + blockIdx.x * blockDim.x + threadIdx.x;  // outputs [t_begin, t_end) of T
    int b = blockIdx.y;
    if (t >= t_end) return;
    const float4* x4 = reinterpret_cast<const float4*>(x) + (size_t)b * (C / 4) * T;
    float acc = 0.f;
#pragma unroll
    for (int cg = 0; cg < C / 4; cg++) {
#pragma unroll
        for (int j = 0; j < K; j++) {
            int tt = t + j - K / 2;
            if (tt >= 0 && tt < T) {
                float4 v = x4[(size_t)cg * T + tt];
                acc = fmaf(lrelu(v.x, slope), sw[(cg * 4 + 0) * K + j], acc);
                acc = fmaf(lrelu(v.y, slope), sw[(cg * 4 + 1) * K + j], acc);
                acc = fmaf(lrelu(v.z, slope), sw[(cg * 4 + 2) * K + j], acc);
                acc = fmaf(lrelu(v.w, slope), sw[(cg * 4 + 3) * K + j], acc);
            }
        }
    }
    y[(size_t)b * T + t] = tanhf(acc);
}

// ------------------------------------------------------------------------------------------------
// Tensor-core attention, middle stage (the Q.K^T and P.V contractions run on wgmma: tc_attn_qk / tc_attn_pv).
// S: c4 over keys [Z = B*heads][Fp/4][T queries][4] holding q_i.k_j; rewritten in place with the softmax
// probabilities of reference attentions.py:280-308 (banded relative-key logits added here, keys >= len excluded,
// rows of invalid queries and columns >= len zeroed so the P.V GEMM can run over the padded key range).
// Also initialises att[b][h*DK+d][i] = sum_r p[i,i+r-w] * Ev[r][d] (relative-value term, :311-318); the P.V GEMM
// then accumulates onto it.  Block = 32 queries x 4 key partitions; loads are coalesced across queries.
// ------------------------------------------------------------------------------------------------
template <int DK, int NP>
__global__ void __launch_bounds__(32 * NP) k_attn_softmax(const float* __restrict__ qkv, float* __restrict__ S, const float* __restrict__ rel_k,
                                                     const float* __restrict__ rel_v, float* __restrict__ att, int H, int heads, int T, int Fp,
                                                     const int* __restrict__ lens, int window) {
    pdl_wait();
    constexpr int NCG = DK / 4;
    __shared__ float sEk[9 * DK], sEv[9 * DK];
    __shared__ float sqrel[NP][32][9];
    __shared__ float sm[NP][32], sl[NP][32];
    __shared__ float sprel[32][9];
    const int tid = threadIdx.x, qi = tid & 31, part = tid >> 5;
    const int z = blockIdx.y, b = z / heads, h = z - b * heads;
    const int i = blockIdx.x * 32 + qi;
    const int len = lens ? lens[b] : T;
    const int nrel = 2 * window + 1;
    for (int k = tid; k < nrel * DK; k += 32 * NP) { sEk[k] = rel_k[k]; sEv[k] = rel_v[k]; }
    for (int k = tid; k < 32 * 9; k += 32 * NP) sprel[k / 9][k % 9] = 0.f;
    __syncthreads();
    const bool inb = i < T, valid = i < len;
    // ---- relative-key logits q_i . Ek[r] (each partition sums NCG/4 channel groups)
    {
        float acc[9];
#pragma unroll
        for (int r = 0; r < 9; r++) acc[r] = 0.f;
        if (inb) {
            const float4* q4 = reinterpret_cast<const float4*>(qkv) + ((size_t)b * (3 * H / 4) + h * NCG) * T + i;
            for (int cg = part; cg < NCG; cg += NP) {
                const float4 qv = q4[(size_t)cg * T];
#pragma unroll
                for (int r = 0; r < 9; r++) {
                    if (r < nrel) {
                        const float* e = &sEk[r * DK + cg * 4];
                        acc[r] = fmaf(qv.x, e[0], fmaf(qv.y, e[1], fmaf(qv.z, e[2], fmaf(qv.w, e[3], acc[r]))));
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < 9; r++) sqrel[part][qi][r] = acc[r];
    }
    __syncthreads();
    float qrel[9];
#pragma unroll
    for (int r = 0; r < 9; r++) { float a = 0.f;
#pragma unroll
        for (int pp = 0; pp < NP; pp++) a += sqrel[pp][qi][r];
        qrel[r] = a; }
    float4* Srow = reinterpret_cast<float4*>(S) + (size_t)z * (Fp / 4) * T + i;
    auto rel_of = [&](int d) { float v = 0.f;
#pragma unroll
        for (int r = 0; r < 9; r++) v = (r == d) ? qrel[r] : v;
        return v; };
    // ---- pass 1: online (max, sum) over this partition's key groups
    float m = -INFINITY, l = 0.f;
    const int ngv = (len + 3) / 4;
    if (valid) {
        // 4 key groups per iteration: the loads are issued together (the online max/sum chain is serial, the loads are not)
        for (int jg0 = part; jg0 < ngv; jg0 += 4 * NP) {
            float4 sv[4];
#pragma unroll
            for (int u = 0; u < 4; u++) if (jg0 + NP * u < ngv) sv[u] = Srow[(size_t)(jg0 + NP * u) * T];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int jg = jg0 + NP * u;
                if (jg >= ngv) break;
                float v[4] = {sv[u].x, sv[u].y, sv[u].z, sv[u].w};
                float mx = -INFINITY;
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int j = jg * 4 + e, d = j - i + window;
                    if ((unsigned)d < (unsigned)nrel) v[e] += rel_of(d);
                    if (j >= len) v[e] = -INFINITY;
                    mx = fmaxf(mx, v[e]);
                }
                if (mx > m) { l *= expf(m - mx); m = mx; }
#pragma unroll
                for (int e = 0; e < 4; e++) l += expf(v[e] - m);
            }
        }
    }
    sm[part][qi] = m; sl[part][qi] = l;
    __syncthreads();
    float M = -INFINITY;
#pragma unroll
    for (int pp = 0; pp < NP; pp++) M = fmaxf(M, sm[pp][qi]);
    float L = 0.f;
#pragma unroll
    for (int pp = 0; pp < NP; pp++) if (sm[pp][qi] > -INFINITY) L += sl[pp][qi] * expf(sm[pp][qi] - M);
    const float inv = (valid && L > 0.f) ? 1.f / L : 0.f;
    // ---- pass 2: probabilities (zeros for excluded keys / invalid queries) over the PADDED key range
    if (inb) {
        for (int jg0 = part; jg0 < Fp / 4; jg0 += 4 * NP) {
            float4 sv[4];
#pragma unroll
            for (int u = 0; u < 4; u++) if (valid && jg0 + NP * u < ngv) sv[u] = Srow[(size_t)(jg0 + NP * u) * T];
#pragma unroll
            for (int u = 0; u < 4; u++) {
                const int jg = jg0 + NP * u;
                if (jg >= Fp / 4) break;
                float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
                if (valid && jg < ngv) {
                    float v[4] = {sv[u].x, sv[u].y, sv[u].z, sv[u].w}, pr[4];
#pragma unroll
                    for (int e = 0; e < 4; e++) {
                        const int j = jg * 4 + e, d = j - i + window;
                        if ((unsigned)d < (unsigned)nrel) v[e] += rel_of(d);
                        pr[e] = (j < len) ? tf32_rna(expf(v[e] - M) * inv) : 0.f;  // TF32-exact: the P.V GEMM skips its prologue
                        if ((unsigned)d < (unsigned)nrel && j < len) sprel[qi][d] = pr[e];
                    }
                    out = make_float4(pr[0], pr[1], pr[2], pr[3]);
                }
                Srow[(size_t)jg * T] = out;
            }
        }
    }
    __syncthreads();
    // ---- relative-value term -> initial value of the attention output
    if (inb) {
        float4* o4 = reinterpret_cast<float4*>(att) + ((size_t)b * (H / 4) + h * NCG) * T + i;
        for (int cg = part; cg < NCG; cg += NP) {
            float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < nrel; r++) {
                const float pw = sprel[qi][r];
                const float* e = &sEv[r * DK + cg * 4];
                o.x = fmaf(pw, e[0], o.x); o.y = fmaf(pw, e[1], o.y); o.z = fmaf(pw, e[2], o.z); o.w = fmaf(pw, e[3], o.w);
            }
            o4[(size_t)cg * T] = o;
        }
    }
}

// V^T pack for the P.V GEMM: vt[z][Fp/32][8][DK][4] (the wgmma K-major B-operand image, K = keys), zeros for keys >= len.
template <int DK>
__global__ void k_pack_vt(const float* __restrict__ qkv, float* __restrict__ vt, int H, int heads, int T, int Fp, const int* __restrict__ lens) {
    pdl_wait();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int cg = blockIdx.y, z = blockIdx.z, b = z / heads, h = z - b * heads;
    if (t >= Fp) return;
    const int len = lens ? lens[b] : T;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t < len && t < T) v = reinterpret_cast<const float4*>(qkv)[((size_t)b * (3 * H / 4) + 2 * H / 4 + h * (DK / 4) + cg) * T + t];
    float* dst = vt + ((((size_t)z * (Fp / 32) + t / 32) * 8 + (t % 32) / 4) * DK + cg * 4) * 4 + (t & 3);
    dst[0] = v.x; dst[4] = v.y; dst[8] = v.z; dst[12] = v.w;
}

__global__ void k_scale_i64(const long long* __restrict__ a, long long* __restrict__ b, int s, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) b[i] = a[i] * s;
}

// 16-bit PCM conversion exactly as gradio.processing_utils.convert_to_16_bit_wav does for float input (called on every
// infer() result by reference webui.py:86, 129, 198): data / abs(data).max() * 32767 -> astype(int16) (truncation), all in
// float32.  Pass 1: per-utterance peak over the valid samples (positive floats order like their bit patterns).
__global__ void k_wave_peak(const float* __restrict__ w, long long L, const long long* __restrict__ nvalid, unsigned* __restrict__ peak) {
    const int b = blockIdx.y;
    const long long n = nvalid ? min(nvalid[b], L) : L;
    float m = 0.f;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(w[(size_t)b * L + t]));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(peak + b, __float_as_uint(m));
}
__global__ void k_wave_to_pcm16(const float* __restrict__ w, long long L, const long long* __restrict__ nvalid, const unsigned* __restrict__ peak,
                                short* __restrict__ out) {
    const int b = blockIdx.y;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= L) return;
    const long long n = nvalid ? min(nvalid[b], L) : L;
    const float pk = __uint_as_float(peak[b]);
    short v = 0;
    if (t < n && pk > 0.f) v = (short)(int)__fmul_rn(__fdiv_rn(w[(size_t)b * L + t], pk), 32767.f);  // C cast = truncation toward zero, as astype(int16)
    out[(size_t)b * L + t] = v;
}


}  // namespace bv2
