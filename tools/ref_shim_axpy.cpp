// ref_shim_axpy.cpp -- extern "C" wrapper around the REFERENCE's naive Axpy oracle, axpy_nv_basic
// (test/saber/test_saber_axpy.cpp:18-52), compiled from the source where it lies (never copied):
// tools/make_ref_axpy_golden.py cuts exactly that function template into ref_axpy.inc next to this file in a temporary
// directory and compiles both with -ffp-contract=off. The reference function reads only num / channel / height / width
// and the data pointers of its tensors, so a minimal Tensor template stands in for saber's. TEST INFRASTRUCTURE: it only
// produces tests/golden/ref_axpy.json.
#include <vector>

template <typename T>
struct Tensor {
    int n, c, h, w;
    float* p;
    int num() const { return n; }
    int channel() const { return c; }
    int height() const { return h; }
    int width() const { return w; }
    const void* data() const { return p; }
    void* mutable_data() { return p; }
};
template <typename T>
struct AxpyParam {};
struct Host {};

#include "ref_axpy.inc"

extern "C" {

// NCHW fp32: scale [n][c] (the gate), x and y [n][c][h][w] -> out [n][c][h][w], in the reference's input order
void ref_axpy_nchw(float* scale, float* x, float* y, float* out, int n, int c, int h, int w) {
    Tensor<Host> ts{n, c, 1, 1, scale}, tx{n, c, h, w, x}, ty{n, c, h, w, y}, to{n, c, h, w, out};
    std::vector<Tensor<Host>*> ins = {&ts, &tx, &ty}, outs = {&to};
    AxpyParam<Host> param;
    axpy_nv_basic<float, Host, Host>(ins, outs, param);
}

}  // extern "C"
