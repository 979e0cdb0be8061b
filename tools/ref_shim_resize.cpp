// ref_shim_resize.cpp -- extern "C" wrapper around the REFERENCE's x86 BILINEAR_NO_ALIGN resize,
// resize_bilinear_no_align_kernel (saber/funcs/impl/x86/saber_resize.cpp:103-153), compiled from the source where it
// lies (never copied): tools/make_ref_resize_golden.py cuts exactly that function template into ref_resize.inc next
// to this file in a temporary directory and compiles both with -ffp-contract=off. TEST INFRASTRUCTURE: it only
// produces tests/golden/ref_resize.json.
#include "ref_resize.inc"

extern "C" {

// uint8 HWC image (h x w x c, read as fp32) -> fp32 HWC image resized to oh x ow, the reference's arithmetic
void ref_resize_bilinear_no_align_hwc(const float* src, int h, int w, int c, float* dst, int oh, int ow) {
    resize_bilinear_no_align_kernel<float>(ow, oh, 1, c, /*dst w, h, channel, batch strides*/ c, ow * c, 1, oh * ow * c,
                                           w, h, /*src strides*/ c, w * c, 1, h * w * c, 0.f, 0.f, src, dst);
}

}  // extern "C"
