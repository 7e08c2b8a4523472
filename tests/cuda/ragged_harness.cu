// Ragged-batch harness: the kernel harness (kernel_harness.cu, included whole) plus one k_g2_conv launch whose items stop at their own
// lengths (G2Epi::lens / lens_scale), loaded by tests/test_ragged_gpu.py through ctypes.  Same buffer conventions as the kernel
// harness: the output sits between two guard regions and the caller supplies its initial contents.
// Built with the product flags by bert_vits2_b200/_lib.py (build_harness(ragged=True)); see tests/ragged_harness.py.
#include "kernel_harness.cu"

extern "C" {

// kh_g2_conv with item b's rows ending at min(T, lens[b] * lens_scale) (lens: HOST [B], frames; lens_scale: M-axis rows per frame)
int kh_g2_conv_ragged(const KhG2Args* a, const int* lens, int lens_scale, void* y, KhG2Plan* plan, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        const int To = a->T * (a->u ? a->u : 1);
        const size_t xb = H8::bytes(a->B, a->Cin, a->T), yb = H8::bytes(a->B, a->Cout, To);
        H8 x = h8_view(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(a->x), xb)), a->B, a->Cin, a->T);
        H8 yy = h8_view(reinterpret_cast<uint4*>(ar.guarded(y, yb)), a->B, a->Cout, To);
        H8 r;
        if (a->res) r = h8_view(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(a->res), yb)), a->B, a->Cout, To);
        const float* dbias = ar.up(a->bias, (size_t)a->Cout);
        const float* dbias_b = ar.up(a->bias_b, (size_t)a->bias_b_elems);
        G2Params p; TcConvW cw;
        const G2Plan pl = g2_plan_of(*a, &ar, x, yy, a->res ? &r : nullptr, dbias, dbias_b, p, cw);
        fill_g2(pl, cw, plan);
        G2Epi e;
        e.res = a->res ? &r : nullptr; e.accumulate = a->accumulate; e.out_scale = a->out_scale; e.bias_b = dbias_b; e.bias_b_stride = a->bias_b_stride;
        e.dil = a->dil ? a->dil : 1; e.st_override = a->st_override;
        e.lens = ar.up(lens, (size_t)a->B); e.lens_scale = lens_scale;
        g2_conv(cw, dbias, x, yy, e, 0, a->num_sms);
        finish(err_flag);
        *guard_ok = read_guarded(reinterpret_cast<const uint8_t*>(yy.p - G2_PADL), y, yb);
    });
}

}  // extern "C"
