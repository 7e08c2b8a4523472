// Ragged-stream harness: the bounded-stream harness (stream_bounded_harness.cu, included whole, with the kernel harness) plus one
// k_g2_conv launch that is a window of a ragged stream (G2Epi::lens / lens_scale / ragged_stream) on tensors held as a resident row
// range, loaded by tests/test_ragged_stream_gpu.py through ctypes.  Same buffer conventions as the kernel harness: the output sits
// between two guard regions and the caller supplies its initial contents.
// Built with the product flags by bert_vits2_b200/_lib.py (build_harness(ragged_stream=True)); see tests/ragged_stream_harness.py.
#include "stream_bounded_harness.cu"

extern "C" {

// kh_g2_conv_resident with item b's rows ending at min(t_end, lens[b] * lens_scale) (lens: HOST [B], frames; lens_scale: M-axis rows
// per frame) and zeros in every row of the window from there on
int kh_g2_conv_ragged_stream(const KhG2Args* a, const int* lens, int lens_scale, int t_begin, int t_end, int x_base, int x_rows, int y_base,
                             int y_rows, int res_base, int res_rows, void* y, int* guard_ok, int* err_flag) {
    return guarded_call([&] {
        init_device();
        Arena ar;
        const int To = a->T * (a->u ? a->u : 1);
        const size_t xb = H8::bytes(a->B, a->Cin, x_rows), yb = H8::bytes(a->B, a->Cout, y_rows);
        H8 x = h8_resident(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(a->x), xb)), a->B, a->Cin, a->T, x_base, x_rows);
        H8 yy = h8_resident(reinterpret_cast<uint4*>(ar.guarded(y, yb)), a->B, a->Cout, To, y_base, y_rows);
        H8 r;
        if (a->res) r = h8_resident(reinterpret_cast<uint4*>(ar.up(static_cast<const uint8_t*>(a->res), H8::bytes(a->B, a->Cout, res_rows))), a->B, a->Cout, To,
                                    res_base, res_rows);
        const float* dbias = ar.up(a->bias, (size_t)a->Cout);
        const float* dbias_b = ar.up(a->bias_b, (size_t)a->bias_b_elems);
        G2Params p; TcConvW cw;
        auto whole = [](H8 t) { t.base = 0; t.Tp = G2_PADL + t.T + G2_PADR; return t; };  // the packing call plans the whole output
        const H8 xw = whole(x), yw = whole(yy), rw = whole(r);
        g2_plan_of(*a, &ar, xw, yw, a->res ? &rw : nullptr, dbias, dbias_b, p, cw);  // packs the weights
        G2Epi e;
        e.res = a->res ? &r : nullptr; e.accumulate = a->accumulate; e.out_scale = a->out_scale; e.bias_b = dbias_b; e.bias_b_stride = a->bias_b_stride;
        e.dil = a->dil ? a->dil : 1; e.st_override = a->st_override; e.t_begin = t_begin; e.t_end = t_end;
        e.lens = ar.up(lens, (size_t)a->B); e.lens_scale = lens_scale; e.ragged_stream = 1;
        g2_conv(cw, dbias, x, yy, e, 0, a->num_sms);
        finish(err_flag);
        *guard_ok = read_guarded(reinterpret_cast<const uint8_t*>(yy.p - G2_PADL), y, yb);
    });
}

}  // extern "C"
