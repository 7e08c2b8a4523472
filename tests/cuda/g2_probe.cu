// Standalone hardware probe for the 16-bit-activation Generator conv kernel (bert_vits2_b200/csrc/tc_gen.cuh): k_g2_conv against a
// CPU conv on the identical f16 operands (plain / residual / MRF-accumulate / polyphase-upsample tails, streamed and resident
// weights, super-tile sizes), halo zeroing, and timings of the Generator's shapes at config 2 (F = 1023 frames).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -DBV2_TUNING -o tests/cuda/g2_probe tests/cuda/g2_probe.cu
// Run:   tests/cuda/g2_probe [perf]
#include <cstdio>
#include <cstdlib>
#include <random>
#include <string>
#include <vector>
#include "../../bert_vits2_b200/csrc/tc_gen.cuh"

using namespace bv2;

static std::vector<void*> g_allocs;
static void* dalloc(size_t bytes) { void* p; cudaMalloc(&p, bytes); g_allocs.push_back(p); return p; }
static float* up(const std::vector<float>& v) {
    void* p = dalloc(std::max<size_t>(v.size(), 4) * 4); cudaMemcpy(p, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
    return (float*)p;
}
static int* g_flag = nullptr;
static int g_timeouts = 0;
static void free_all() {
    for (void* p : g_allocs) cudaFree(p);
    g_allocs.clear();
    if (g_flag && *g_flag) { printf("  ^^^ BARRIER TIMEOUT raised by this case\n"); *g_flag = 0; tc_clear_error(); g_timeouts++; }
}
static float h2f(uint16_t u) { __half h; std::memcpy(&h, &u, 2); return __half2float(h); }
static float lre(float v) { return v > 0 ? v : 0.1f * v; }
static float unl(float a) { return a >= 0 ? a : 10.f * a; }

// device H8 tensor filled with NaN patterns, data rows from `vals` ([B][C][T], already f16-representable), halos zeroed by the kernel under test
static H8 make_h8(const std::vector<float>* vals, int B, int C, int T) {
    H8 t; t.B = B; t.C = C; t.T = T; t.Tp = G2_PADL + T + G2_PADR;
    const size_t n = (size_t)B * (C / 8) * t.Tp * 8;
    std::vector<uint16_t> h(n, 0x7e00);  // NaN everywhere
    if (vals)
        for (int b = 0; b < B; b++) for (int c = 0; c < C; c++) for (int tt = 0; tt < T; tt++)
            h[(((size_t)b * (C / 8) + c / 8) * t.Tp + G2_PADL + tt) * 8 + (c & 7)] = f16_rn_host((*vals)[((size_t)b * C + c) * T + tt]);
    uint16_t* d = (uint16_t*)dalloc(n * 2);
    cudaMemcpy(d, h.data(), n * 2, cudaMemcpyHostToDevice);
    t.p = reinterpret_cast<uint4*>(d) + G2_PADL;
    G2HaloList l{}; l.n = 1; l.p[0] = t.p; l.cg_rows[0] = B * (C / 8); l.T[0] = T; l.Tp[0] = t.Tp;
    k_g2_zero_halo<<<dim3(8, 1), 128>>>(l);
    return t;
}
static std::vector<float> read_h8(const H8& t) {
    const size_t n = (size_t)t.B * (t.C / 8) * t.Tp * 8;
    std::vector<uint16_t> h(n);
    cudaMemcpy(h.data(), reinterpret_cast<uint16_t*>(t.p - G2_PADL), n * 2, cudaMemcpyDeviceToHost);
    std::vector<float> o((size_t)t.B * t.C * t.T);
    for (int b = 0; b < t.B; b++) for (int c = 0; c < t.C; c++) for (int tt = 0; tt < t.T; tt++)
        o[((size_t)b * t.C + c) * t.T + tt] = h2f(h[(((size_t)b * (t.C / 8) + c / 8) * t.Tp + G2_PADL + tt) * 8 + (c & 7)]);
    return o;
}
static void f16ify(std::vector<float>& v) { for (auto& x : v) x = f16_round_host(x); }

static int run_conv(int Cin, int Cout, int K, int dil, int T, int B, bool res, bool acc, float scale, int st, int iters) {
    std::mt19937 rng(Cin * 131 + Cout * 17 + K * 7 + dil + T);
    std::normal_distribution<float> nd(0.f, 1.f);
    std::vector<float> x((size_t)B * Cin * T), w((size_t)Cout * Cin * K), bias(Cout), r((size_t)B * Cout * T), y0((size_t)B * Cout * T);
    for (auto& v : x) v = lre(nd(rng));
    for (auto& v : w) v = nd(rng) / std::sqrt((float)(Cin * K));
    for (auto& v : bias) v = nd(rng);
    for (auto& v : r) v = lre(nd(rng));
    for (auto& v : y0) v = lre(nd(rng));
    f16ify(x); f16ify(r); f16ify(y0);
    std::function<float*(const std::vector<float>&)> upf = up;
    TcConvW tw = tc_pack_weights(upf, w, Cout, Cin, K, g2_nt(Cout), 1, g2_kc(Cin));
    H8 hx = make_h8(&x, B, Cin, T), hy = make_h8(acc ? &y0 : nullptr, B, Cout, T), hr = make_h8(&r, B, Cout, T);
    float* dbias = up(bias);
    G2Epi e; e.res = res ? &hr : nullptr; e.accumulate = acc; e.out_scale = scale; e.dil = dil; e.st_override = st;
    g2_conv(tw, dbias, hx, hy, e, 0, 148);
    cudaError_t er = cudaDeviceSynchronize();
    if (er != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(er)); return 1; }
    std::vector<float> got = read_h8(hy);
    const int pad = (K - 1) / 2 * dil;
    std::vector<float> wr(w.size());
    for (size_t i = 0; i < w.size(); i++) wr[i] = f16_round_host(w[i]);
    std::vector<int> ts;
    for (int t = 0; t < T; t += std::max(1, T / 200 - 1)) ts.push_back(t);
    for (int t : {1, 2, 127, 128, 129, 255, 256, 511, 512, 513, T - 2, T - 1}) if (t >= 0 && t < T) ts.push_back(t);
    double maxerr = 0, maxref = 0; int nan = 0;
    for (int b = 0; b < B; b++)
        for (int co = 0; co < Cout; co += (Cout > 64 ? 3 : 1))
            for (int t : ts) {
                double s = bias[co];
                for (int ci = 0; ci < Cin; ci++)
                    for (int j = 0; j < K; j++) {
                        int tt = t + j * dil - pad;
                        if (tt >= 0 && tt < T) s += (double)x[((size_t)b * Cin + ci) * T + tt] * wr[((size_t)co * Cin + ci) * K + j];
                    }
                if (res) s += unl(r[((size_t)b * Cout + co) * T + t]);
                if (acc) s += unl(y0[((size_t)b * Cout + co) * T + t]);
                s = lre((float)(s * scale));
                double g = got[((size_t)b * Cout + co) * T + t];
                if (g != g) nan++;
                maxerr = std::max(maxerr, std::fabs(g - s)); maxref = std::max(maxref, std::fabs(s));
            }
    float ms = 0;
    if (iters > 0) {
        cudaEvent_t a, c; cudaEventCreate(&a); cudaEventCreate(&c);
        e.accumulate = 0;
        e.dbg_skip_wcommit = getenv("G2_SKIP_WCOMMIT") ? 1 : 0;
        e.dbg_flags = getenv("G2_DBG") ? atoi(getenv("G2_DBG")) : 0;
        if (getenv("G2_PROF")) {  // per-CTA phase timeline of the last of three back-to-back launches
            long long* dprof = (long long*)dalloc(4096 * 16 * 8);
            cudaMemset(dprof, 0, 4096 * 16 * 8);
            for (int i = 0; i < 3; i++) { e.prof = i == 2 ? dprof : nullptr; g2_conv(tw, dbias, hx, hy, e, 0, 148); }
            e.prof = nullptr;
            cudaDeviceSynchronize();
            std::vector<long long> hp(4096 * 16);
            cudaMemcpy(hp.data(), dprof, hp.size() * 8, cudaMemcpyDeviceToHost);
            long long t0 = 0; int n = 0;
            for (int i = 0; i < 4096; i++) if (hp[i * 16]) { n++; if (!t0 || hp[i * 16] < t0) t0 = hp[i * 16]; }
            printf("  prof (%d CTAs; ns since first CTA start): cta: start | pdl-wait begin/end | first A | mma issue end | acc0 full | accN full | tail end || clk waitA waitW\n", n);
            for (int i : {0, 1, n / 2, n - 1}) {
                const long long* q = &hp[(size_t)i * 16];
                printf("   cta %4d: %6lld | %6lld %6lld | %6lld | %6lld | %6lld | %6lld | %6lld || %8lld %8lld || mma phase %lld clk for %lld MMAs = %.1f clk/MMA, %.2f GHz\n", i, q[0] - t0, q[1] - t0, q[2] - t0, q[3] - t0, q[4] - t0, q[5] - t0, q[6] - t0, q[7] - t0, q[8], q[9],
                       q[11] - q[10], q[12], (double)(q[11] - q[10]) / (double)std::max(1ll, q[12]), (double)(q[11] - q[10]) / (double)std::max(1ll, q[4] - q[3]));
            }
        }
        for (int i = 0; i < 3; i++) g2_conv(tw, dbias, hx, hy, e, 0, 148);
        cudaEventRecord(a);
        for (int i = 0; i < iters; i++) g2_conv(tw, dbias, hx, hy, e, 0, 148);
        cudaEventRecord(c); cudaEventSynchronize(c); cudaEventElapsedTime(&ms, a, c); ms /= iters;
    }
    double flop = 2.0 * B * T * (double)Cin * Cout * K;
    double bytes = 2.0 * B * T * (Cin + Cout * (1 + (res ? 1 : 0)));
    bool ok = nan == 0 && maxerr < 4e-3 * std::max(1.0, maxref);  // f16 output rounding: 2^-11 relative
    printf("%s G2 Cin=%3d Cout=%3d K=%2d dil=%d T=%6d B=%d res=%d acc=%d st=%d : maxerr %.3e (ref max %.2f, nan %d)", ok ? "PASS" : "FAIL", Cin, Cout, K, dil, T, B,
           (int)res, (int)acc, st, maxerr, maxref, nan);
    if (iters > 0) printf("  | %.4f ms  %.1f TFLOP/s  %.0f GB/s(f16)", ms, flop / ms * 1e-9, bytes / ms * 1e-6);
    printf("\n"); fflush(stdout);
    free_all();
    return ok ? 0 : 1;
}

static int run_ups(int Cin, int Cout, int K, int u, int T, int B, int iters) {
    std::mt19937 rng(Cin * 13 + Cout + K + u + T);
    std::normal_distribution<float> nd(0.f, 1.f);
    const int To = T * u, p = (K - u) / 2;
    std::vector<float> x((size_t)B * Cin * T), w((size_t)Cin * Cout * K), bias(Cout);
    for (auto& v : x) v = lre(nd(rng));
    for (auto& v : w) v = nd(rng) / std::sqrt((float)(Cin * K / u));
    for (auto& v : bias) v = nd(rng);
    f16ify(x);
    std::function<float*(const std::vector<float>&)> upf = up;
    TcConvW tw = tc_pack_upsample(upf, w, Cin, Cout, K, u, g2_kc(Cin), 1, true, 128);
    H8 hx = make_h8(&x, B, Cin, T), hy = make_h8(nullptr, B, Cout, To);
    float* dbias = up(bias);
    g2_conv(tw, dbias, hx, hy, G2Epi(), 0, 148);
    cudaError_t er = cudaDeviceSynchronize();
    if (er != cudaSuccess) { printf("CUDA error: %s\n", cudaGetErrorString(er)); return 1; }
    std::vector<float> got = read_h8(hy);
    double maxerr = 0, maxref = 0; int nan = 0;
    for (int b = 0; b < B; b++)
        for (int co = 0; co < Cout; co += 3)
            for (int n = 0; n < To; n += std::max(1, To / 300)) {
                double s = bias[co];
                for (int i = 0; i < T; i++) {
                    int j = n + p - i * u;
                    if (j < 0 || j >= K) continue;
                    for (int ci = 0; ci < Cin; ci++) s += (double)x[((size_t)b * Cin + ci) * T + i] * f16_round_host(w[((size_t)ci * Cout + co) * K + j]);
                }
                s = lre((float)s);
                double g = got[((size_t)b * Cout + co) * To + n];
                if (g != g) nan++;
                maxerr = std::max(maxerr, std::fabs(g - s)); maxref = std::max(maxref, std::fabs(s));
            }
    float ms = 0;
    if (iters > 0) {
        cudaEvent_t a, c; cudaEventCreate(&a); cudaEventCreate(&c);
        for (int i = 0; i < 3; i++) g2_conv(tw, dbias, hx, hy, G2Epi(), 0, 148);
        cudaEventRecord(a);
        for (int i = 0; i < iters; i++) g2_conv(tw, dbias, hx, hy, G2Epi(), 0, 148);
        cudaEventRecord(c); cudaEventSynchronize(c); cudaEventElapsedTime(&ms, a, c); ms /= iters;
    }
    bool ok = nan == 0 && maxerr < 4e-3 * std::max(1.0, maxref);
    printf("%s G2 UPS Cin=%3d Cout=%3d K=%2d u=%d T=%6d B=%d (Kp=%d) : maxerr %.3e (ref max %.2f, nan %d)", ok ? "PASS" : "FAIL", Cin, Cout, K, u, T, B, tw.K, maxerr, maxref, nan);
    if (iters > 0) printf("  | %.4f ms", ms);
    printf("\n"); fflush(stdout);
    free_all();
    return ok ? 0 : 1;
}

int main(int argc, char** argv) {
    const bool perf = argc > 1;
    g_flag = tc_init_device();
    g2_init_device();
    int fails = 0;
    if (argc > 1 && std::string(argv[1]) == "case") {  // g2_probe case Cin Cout K dil T st iters res [more cases ...]
        for (int a = 2; a + 7 < argc; a += 8) {
            run_conv(atoi(argv[a]), atoi(argv[a + 1]), atoi(argv[a + 2]), atoi(argv[a + 3]), atoi(argv[a + 4]), 1, atoi(argv[a + 7]) != 0, false, 1.f, atoi(argv[a + 5]), atoi(argv[a + 6]));
        }
        return 0;
    }
    // ---- correctness: small shapes, every tail, edge tiles, both weight modes
    fails += run_conv(16, 16, 3, 1, 300, 1, false, false, 1.f, 0, 0);
    fails += run_conv(16, 16, 11, 5, 1000, 2, true, false, 1.f, 0, 0);
    fails += run_conv(16, 16, 7, 3, 5000, 1, true, true, 1.f / 3, 0, 0);      // resident, several m-groups
    fails += run_conv(32, 32, 11, 5, 3000, 1, true, false, 1.f, 0, 0);
    fails += run_conv(32, 32, 3, 1, 129, 3, true, true, 1.f, 0, 0);
    fails += run_conv(64, 64, 7, 3, 2000, 1, true, false, 1.f, 0, 0);          // streamed, KC = 16
    fails += run_conv(64, 64, 11, 1, 700, 2, false, false, 1.f, 3, 0);
    fails += run_conv(128, 128, 3, 1, 1000, 1, true, false, 1.f, 4, 0);        // streamed, KC = 32, MG = 4
    fails += run_conv(128, 128, 11, 5, 600, 1, true, true, 1.f / 3, 2, 0);
    fails += run_conv(256, 256, 7, 3, 500, 1, true, false, 1.f, 2, 0);         // two N tiles
    fails += run_conv(192, 512, 7, 1, 300, 2, false, false, 1.f, 0, 0);        // conv_pre shape
    fails += run_ups(512, 256, 16, 8, 200, 1, 0);
    fails += run_ups(128, 64, 8, 2, 700, 2, 0);
    fails += run_ups(32, 16, 8, 2, 3000, 1, 0);
    printf("G2 PROBE correctness: %d failure(s), %d barrier timeout(s)\n", fails, g_timeouts);
    if (perf && fails == 0 && g_timeouts == 0) {
        const int F = 1023;
        printf("---- Generator shapes at F = %d frames (config 2)\n", F);
        run_conv(192, 512, 7, 1, F, 1, false, false, 1.f, 0, 20);
        run_ups(512, 256, 16, 8, F, 1, 20);
        int ch = 256, L = F * 8;
        const int us[5] = {8, 8, 2, 2, 2}, uk[5] = {16, 16, 8, 8, 8};
        for (int i = 0; i < 5; i++) {
            if (i > 0) { run_ups(ch * 2, ch, uk[i], us[i], L, 1, 20); L *= us[i]; }
            for (int K : {3, 7, 11}) {
                run_conv(ch, ch, K, 1, L, 1, false, false, 1.f, 0, 20);
                run_conv(ch, ch, K, 5, L, 1, true, false, 1.f, 0, 20);
            }
            ch /= 2;
        }
        printf("---- super-tile sweep (stage 1: C = 128, stage 0: C = 256, stage 2: C = 64)\n");
        for (int st : {1, 2, 3, 4}) run_conv(128, 128, 7, 1, 65472, 1, true, false, 1.f, st, 20);
        for (int st : {1, 2, 4}) run_conv(256, 256, 7, 1, 8184, 1, true, false, 1.f, st, 20);
        for (int st : {2, 4, 7, 8}) run_conv(64, 64, 7, 1, 130944, 1, true, false, 1.f, st, 20);
    }
    printf("G2 PROBE done: %d failure(s), %d barrier timeout(s)\n", fails, g_timeouts);
    return fails || g_timeouts ? 1 : 0;
}
