// Standalone timing probe for the 16-bit-activation Generator conv kernel (bert_vits2_b200/csrc/tc_gen.cuh): k_g2_conv at the
// Generator's shapes at config 2 (F = 1023 frames), super-tile sweeps, and per-CTA phase timelines (G2_PROF=1).  Correctness of the
// kernel is checked by tests/test_kernels_gpu.py (every tail, both weight modes, every super-tile size, halo zeroing, full outputs).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -DBV2_TUNING -o tests/cuda/g2_probe tests/cuda/g2_probe.cu
// Run:   tests/cuda/g2_probe                                   (Generator shapes + super-tile sweep)
//        tests/cuda/g2_probe case Cin Cout K dil T st iters res [more cases ...]
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

// device H8 tensor (random f16 activations, zero halos)
static H8 make_h8(int B, int C, int T, std::mt19937& rng) {
    H8 t; t.B = B; t.C = C; t.T = T; t.Tp = G2_PADL + T + G2_PADR;
    const size_t n = (size_t)B * (C / 8) * t.Tp * 8;
    std::normal_distribution<float> nd(0.f, 1.f);
    std::vector<uint16_t> h(n, 0);
    for (int b = 0; b < B; b++) for (int g = 0; g < C / 8; g++) for (int tt = 0; tt < T; tt++) for (int e = 0; e < 8; e++) {
        const float v = nd(rng);
        h[(((size_t)b * (C / 8) + g) * t.Tp + G2_PADL + tt) * 8 + e] = f16_rn_host(v > 0 ? v : 0.1f * v);
    }
    uint16_t* d = (uint16_t*)dalloc(n * 2);
    cudaMemcpy(d, h.data(), n * 2, cudaMemcpyHostToDevice);
    t.p = reinterpret_cast<uint4*>(d) + G2_PADL;
    return t;
}

static float time_launches(const std::function<void()>& f, int iters) {
    cudaEvent_t a, c; cudaEventCreate(&a); cudaEventCreate(&c);
    for (int i = 0; i < 3; i++) f();
    cudaEventRecord(a);
    for (int i = 0; i < iters; i++) f();
    cudaEventRecord(c); cudaEventSynchronize(c);
    float ms = 0; cudaEventElapsedTime(&ms, a, c);
    cudaEventDestroy(a); cudaEventDestroy(c);
    return ms / iters;
}

static void run_conv(int Cin, int Cout, int K, int dil, int T, int B, bool res, int st, int iters) {
    std::mt19937 rng(Cin * 131 + Cout * 17 + K * 7 + dil + T);
    std::normal_distribution<float> nd(0.f, 1.f);
    std::vector<float> w((size_t)Cout * Cin * K), bias(Cout);
    for (auto& v : w) v = nd(rng) / std::sqrt((float)(Cin * K));
    for (auto& v : bias) v = nd(rng);
    std::function<float*(const std::vector<float>&)> upf = up;
    TcConvW tw = tc_pack_weights(upf, w, Cout, Cin, K, g2_nt(Cout), 1, g2_kc(Cin));
    H8 hx = make_h8(B, Cin, T, rng), hy = make_h8(B, Cout, T, rng), hr = make_h8(B, Cout, T, rng);
    float* dbias = up(bias);
    G2Epi e; e.res = res ? &hr : nullptr; e.dil = dil; e.st_override = st;
    e.dbg_skip_wcommit = getenv("G2_SKIP_WCOMMIT") ? 1 : 0;
    e.dbg_flags = getenv("G2_DBG") ? atoi(getenv("G2_DBG")) : 0;
    if (getenv("G2_PROF")) {  // per-CTA phase timeline of the last of three back-to-back launches
        long long* dprof = (long long*)dalloc(4096 * 16 * 8);
        cudaMemset(dprof, 0, 4096 * 16 * 8);
        for (int i = 0; i < 3; i++) { e.prof = i == 2 ? dprof : nullptr; g2_conv(tw, dbias, hx, hy, e, 0, 132); }
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
    const float ms = time_launches([&] { g2_conv(tw, dbias, hx, hy, e, 0, 132); }, iters);
    const double flop = 2.0 * B * T * (double)Cin * Cout * K, bytes = 2.0 * B * T * (Cin + Cout * (1 + (res ? 1 : 0)));
    printf("G2 Cin=%3d Cout=%3d K=%2d dil=%d T=%6d B=%d res=%d st=%d : %.4f ms  %.1f TFLOP/s  %.0f GB/s(f16)\n", Cin, Cout, K, dil, T, B, (int)res, st,
           ms, flop / ms * 1e-9, bytes / ms * 1e-6);
    fflush(stdout);
    free_all();
}

static void run_ups(int Cin, int Cout, int K, int u, int T, int B, int iters) {
    std::mt19937 rng(Cin * 13 + Cout + K + u + T);
    std::normal_distribution<float> nd(0.f, 1.f);
    std::vector<float> w((size_t)Cin * Cout * K), bias(Cout);
    for (auto& v : w) v = nd(rng) / std::sqrt((float)(Cin * K / u));
    for (auto& v : bias) v = nd(rng);
    std::function<float*(const std::vector<float>&)> upf = up;
    TcConvW tw = tc_pack_upsample(upf, w, Cin, Cout, K, u, g2_kc(Cin), 1, true, 128);
    H8 hx = make_h8(B, Cin, T, rng), hy = make_h8(B, Cout, T * u, rng);
    float* dbias = up(bias);
    const float ms = time_launches([&] { g2_conv(tw, dbias, hx, hy, G2Epi(), 0, 132); }, iters);
    printf("G2 UPS Cin=%3d Cout=%3d K=%2d u=%d T=%6d B=%d (Kp=%d) : %.4f ms\n", Cin, Cout, K, u, T, B, tw.K, ms);
    fflush(stdout);
    free_all();
}

int main(int argc, char** argv) {
    g_flag = tc_init_device();
    g2_init_device();
    if (argc > 1 && std::string(argv[1]) == "case") {  // g2_probe case Cin Cout K dil T st iters res [more cases ...]
        for (int a = 2; a + 7 < argc; a += 8)
            run_conv(atoi(argv[a]), atoi(argv[a + 1]), atoi(argv[a + 2]), atoi(argv[a + 3]), atoi(argv[a + 4]), 1, atoi(argv[a + 7]) != 0,
                     atoi(argv[a + 5]), atoi(argv[a + 6]));
        return g_timeouts ? 1 : 0;
    }
    const int F = 1023;
    printf("---- Generator shapes at F = %d frames (config 2)\n", F);
    run_conv(192, 512, 7, 1, F, 1, false, 0, 20);
    run_ups(512, 256, 16, 8, F, 1, 20);
    int ch = 256, L = F * 8;
    const int us[5] = {8, 8, 2, 2, 2}, uk[5] = {16, 16, 8, 8, 8};
    for (int i = 0; i < 5; i++) {
        if (i > 0) { run_ups(ch * 2, ch, uk[i], us[i], L, 1, 20); L *= us[i]; }
        for (int K : {3, 7, 11}) {
            run_conv(ch, ch, K, 1, L, 1, false, 0, 20);
            run_conv(ch, ch, K, 5, L, 1, true, 0, 20);
        }
        ch /= 2;
    }
    printf("---- super-tile sweep (stage 1: C = 128, stage 0: C = 256, stage 2: C = 64)\n");
    for (int st : {1, 2, 3, 4}) run_conv(128, 128, 7, 1, 65472, 1, true, st, 20);
    for (int st : {1, 2, 4}) run_conv(256, 256, 7, 1, 8184, 1, true, st, 20);
    for (int st : {2, 4, 7, 8}) run_conv(64, 64, 7, 1, 130944, 1, true, st, 20);
    printf("G2 PROBE done: %d barrier timeout(s)\n", g_timeouts);
    return g_timeouts ? 1 : 0;
}
