// Resize + centre crop of 8-bit images of any size to the image input's H x W, on the GPU (include/b200_saber.h has
// the geometry and the arithmetic of every filter). The per-image sizes live in a device table the host fills per
// request, so the launches depend only on (n, c, H, W) (and, for the Pillow filters, the workspace's max_h, max_w and
// resize_short) and the op is captured once into the Net's CUDA graph.
//
// Replaces (reference): the host-side preprocessing of test/framework/net/classification_accuracy.cpp and the x86
// BILINEAR_NO_ALIGN resize, saber/funcs/impl/x86/saber_resize.cpp:103-153 (resize_bilinear_no_align_kernel), whose
// fp32 result this kernel reproduces bit for bit before rounding to 8 bits.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200_saber.h"
#include "common.cuh"
#include "ptx.cuh"
#include "vec.cuh"

namespace b200 {

namespace {

constexpr int kResizeThreads = 256;
constexpr int kPixelsPerThread = 4;         // a run of 4 output pixels of one row: 4*C bytes, C 32-bit words
constexpr long long kMaxResized = 1ll << 23;

// One axis of the source coordinate: f = max(scale * ((float)r + 0.5f) - 0.5f, 0), taps i0, i1 and the fraction
// f - i0; every fp32 step rounded on its own, as the reference computes it without contraction.
struct Axis {
    int i0, i1;
    float f;
};
__device__ __forceinline__ Axis resize_axis(float scale, int r, int size) {
    float f = __fsub_rn(__fmul_rn(scale, __fadd_rn(static_cast<float>(r), 0.5f)), 0.5f);
    f = f < 0.f ? 0.f : f;
    Axis a;
    a.i0 = static_cast<int>(f);
    a.i1 = a.i0 + (a.i0 < size - 1 ? 1 : 0);
    a.f = __fsub_rn(f, static_cast<float>(a.i0));
    return a;
}

// ---------------------------------------------------------------------------------------------- table entries
// A kernel reads its table through one of two entry types. b200_image_resize_entry_t is a whole image: the box is the
// frame, at origin (0, 0). b200_image_crop_entry_t is a box of a larger frame; its resize part holds the box's size and
// geometry, so every axis, tap and pass-order rule below runs on the box, and only the source layout sees the frame.
__device__ __forceinline__ const b200_image_resize_entry_t* resize_entry(const b200_image_resize_entry_t* t, int i) {
    return t + i;
}
__device__ __forceinline__ const b200_image_resize_entry_t* resize_entry(const b200_image_crop_entry_t* t, int i) {
    return &t[i].r;
}

// Where a box lies in its frame. h, w: the entry's own (box) size, already loaded.
struct Box {
    int frame_h, frame_w, top, left;
};
__device__ __forceinline__ Box box_of(const b200_image_resize_entry_t*, int h, int w) { return {h, w, 0, 0}; }
__device__ __forceinline__ Box box_of(const b200_image_crop_entry_t* e, int, int) {
    return {__ldg(&e->frame_h), __ldg(&e->frame_w), __ldg(&e->box_top), __ldg(&e->box_left)};
}

// ---------------------------------------------------------------------------------------------- source layouts
// A source layout turns (box, row, column) into the channel bytes of one tap, so the resize kernels read any 8-bit
// layout at tap fetch. `row` is computed once per source row a thread reads; `tap` gives one channel of one pixel.
// Rows and columns are box coordinates: row(y) is frame row top + y, pixel(r, x) frame column left + x.

// Interleaved pixels: frame_h rows of frame_w * C bytes; `img` points at the box's first pixel.
template <int C>
struct Interleaved {
    static constexpr int kChannels = C;
    const uint8_t* img;
    int w;      // the frame's row length in pixels
    __device__ __forceinline__ Interleaved(const uint8_t* frame, const Box& b)
        : img(frame + (static_cast<long long>(b.top) * b.frame_w + b.left) * C), w(b.frame_w) {}
    // the box of table entry i, loading only what this layout reads
    template <class Entry>
    __device__ __forceinline__ static Interleaved at(const uint8_t* src, const Entry* table, int i) {
        const b200_image_resize_entry_t* e = resize_entry(table, i);
        const uint8_t* frame = src + __ldg(&e->offset);
        return Interleaved(frame, box_of(table + i, 0, __ldg(&e->w)));     // frame_h is never read here
    }
    __device__ __forceinline__ const uint8_t* row(int y) const { return img + static_cast<long long>(y) * w * C; }
    __device__ __forceinline__ const uint8_t* pixel(const uint8_t* r, int x) const { return r + x * C; }
    __device__ __forceinline__ uint8_t tap(const uint8_t* p, int ch) const { return __ldg(p + ch); }
};

// OpenCV's COLOR_YUV2RGB_NV12 / _I420 (BT.601 limited range, 20-bit fixed point) of one (Y, U, V) triple, in R, G, B.
__device__ __forceinline__ int yuv_sat8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }
__device__ __forceinline__ int yuv_channel(int Y, int U, int V, int ch) {
    const int yy = (Y > 16 ? Y - 16 : 0) * 1220542 + (1 << 19);
    const int u = U - 128, v = V - 128;
    if (ch == 0) return yuv_sat8((yy + 1673527 * v) >> 20);
    if (ch == 1) return yuv_sat8((yy - 852492 * v - 409993 * u) >> 20);
    return yuv_sat8((yy + 2116026 * u) >> 20);
}

// YUV 4:2:0 (frame_h and frame_w even): the frame_h x frame_w Y plane, then NV12's frame_h/2 rows of frame_w
// interleaved U,V bytes or I420's (frame_h/2) x (frame_w/2) U plane followed by its V plane. Frame pixel (fy, fx) takes
// chroma sample (fy/2, fx/2), so a box at an odd offset or of an odd size reads the chroma blocks it straddles. Every
// channel of a tap reads the same three bytes; once the kernel is unrolled the compiler loads and converts them once
// per tap.
template <int F>
struct Yuv420 {
    static_assert(F == B200_IMAGE_YUV_NV12 || F == B200_IMAGE_YUV_I420, "NV12 or I420");
    static constexpr int kChannels = 3;
    struct Row {
        const uint8_t *y, *u, *v;
    };
    const uint8_t* img;
    Box b;
    __device__ __forceinline__ Yuv420(const uint8_t* frame, const Box& b_) : img(frame), b(b_) {}
    template <class Entry>
    __device__ __forceinline__ static Yuv420 at(const uint8_t* src, const Entry* table, int i) {
        const b200_image_resize_entry_t* e = resize_entry(table, i);
        return Yuv420(src + __ldg(&e->offset), box_of(table + i, __ldg(&e->h), __ldg(&e->w)));
    }
    __device__ __forceinline__ Row row(int y) const {
        const int h = b.frame_h, w = b.frame_w, fy = b.top + y;
        const uint8_t* chroma = img + static_cast<long long>(h) * w;
        Row r;
        r.y = img + static_cast<long long>(fy) * w;
        if constexpr (F == B200_IMAGE_YUV_NV12) {
            r.u = chroma + static_cast<long long>(fy >> 1) * w;
            r.v = r.u + 1;
        } else {
            r.u = chroma + static_cast<long long>(fy >> 1) * (w >> 1);
            r.v = r.u + static_cast<long long>(h >> 1) * (w >> 1);
        }
        return r;
    }
    __device__ __forceinline__ Row pixel(const Row& r, int x) const {
        const int fx = b.left + x;
        const int cx = F == B200_IMAGE_YUV_NV12 ? (fx & ~1) : (fx >> 1);
        return {r.y + fx, r.u + cx, r.v + cx};
    }
    __device__ __forceinline__ int tap(const Row& p, int ch) const {
        return yuv_channel(__ldg(p.y), __ldg(p.u), __ldg(p.v), ch);
    }
};

// Thread = kPixelsPerThread consecutive output pixels of one row of one image. The row's source taps and weights are
// computed once; the 4 taps x C channels of each pixel are read through the read-only path. VEC (out_w % 4 == 0):
// the run is C aligned 32-bit words, stored as one 4-, 8-, 12- or 16-byte write; otherwise byte stores.
template <class Src, class Entry, bool VEC>
__global__ void __launch_bounds__(kResizeThreads) image_resize_kernel(const uint8_t* __restrict__ src,
                                                                      const Entry* __restrict__ table,
                                                                      uint8_t* __restrict__ out, int out_h, int out_w,
                                                                      int runs, long long total) {
    constexpr int C = Src::kChannels;
    pdl_enter();      // the previous request's readers of `out` are done
    const long long t = blockIdx.x * 1ll * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int run = static_cast<int>(t % runs);
    const long long row = t / runs;
    const int y = static_cast<int>(row % out_h);
    const int img = static_cast<int>(row / out_h);
    const b200_image_resize_entry_t* e = resize_entry(table, img);
    const long long offset = __ldg(&e->offset);
    const int h = __ldg(&e->h), w = __ldg(&e->w);
    const int rh = __ldg(&e->rh), rw = __ldg(&e->rw);
    const int top = __ldg(&e->top), left = __ldg(&e->left);

    const Axis ay = resize_axis(__fdiv_rn(static_cast<float>(h), static_cast<float>(rh)), y + top, h);
    const double ry = __dsub_rn(1.0, static_cast<double>(ay.f));
    const Src s(src + offset, box_of(table + img, h, w));
    const auto r0 = s.row(ay.i0);
    const auto r1 = s.row(ay.i1);
    const float sx = __fdiv_rn(static_cast<float>(w), static_cast<float>(rw));
    const int x_begin = run * kPixelsPerThread;
    uint8_t* o = out + ((static_cast<long long>(img) * out_h + y) * out_w + x_begin) * C;

    uint32_t words[C];
#pragma unroll
    for (int i = 0; i < C; ++i) words[i] = 0;
#pragma unroll
    for (int p = 0; p < kPixelsPerThread; ++p) {
        if (!VEC && x_begin + p >= out_w) break;
        const Axis ax = resize_axis(sx, x_begin + p + left, w);
        const double rx = __dsub_rn(1.0, static_cast<double>(ax.f));
        const float w00 = __double2float_rn(__dmul_rn(ry, rx));
        const float w01 = __double2float_rn(__dmul_rn(static_cast<double>(ax.f), ry));
        const float w10 = __double2float_rn(__dmul_rn(static_cast<double>(ay.f), rx));
        const float w11 = __double2float_rn(__dmul_rn(static_cast<double>(ax.f), static_cast<double>(ay.f)));
        const auto q00 = s.pixel(r0, ax.i0), q01 = s.pixel(r0, ax.i1);
        const auto q10 = s.pixel(r1, ax.i0), q11 = s.pixel(r1, ax.i1);
#pragma unroll
        for (int ch = 0; ch < C; ++ch) {
            const float p00 = s.tap(q00, ch), p01 = s.tap(q01, ch);
            const float p10 = s.tap(q10, ch), p11 = s.tap(q11, ch);
            float v = __fadd_rn(__fmul_rn(w00, p00), __fmul_rn(w01, p01));
            v = __fadd_rn(v, __fmul_rn(w10, p10));
            v = __fadd_rn(v, __fmul_rn(w11, p11));
            const uint32_t b = cvt_q8(v, true);
            if constexpr (VEC) {
                const int byte = p * C + ch;
                words[byte >> 2] |= b << (8 * (byte & 3));
            } else {
                o[p * C + ch] = static_cast<uint8_t>(b);
            }
        }
    }
    if constexpr (VEC) {
        if constexpr (C == 4) *reinterpret_cast<uint4*>(o) = make_uint4(words[0], words[1], words[2], words[3]);
        else if constexpr (C == 2) *reinterpret_cast<uint2*>(o) = make_uint2(words[0], words[1]);
        else if constexpr (C == 3) {
            uint32_t* o32 = reinterpret_cast<uint32_t*>(o);
            o32[0] = words[0]; o32[1] = words[1]; o32[2] = words[2];
        } else *reinterpret_cast<uint32_t*>(o) = words[0];
    }
}

template <class Src, class Entry = b200_image_resize_entry_t>
int launch_resize(const b200_image_resize_desc_t* d, const uint8_t* src, const void* table, uint8_t* out,
                  void* stream) {
    const int runs = (d->out_w + kPixelsPerThread - 1) / kPixelsPerThread;
    const long long total = 1ll * d->n * d->out_h * runs;
    const unsigned grid = static_cast<unsigned>((total + kResizeThreads - 1) / kResizeThreads);
    const auto* tab = static_cast<const Entry*>(table);
    const bool vec = d->out_w % kPixelsPerThread == 0;
    return launch("image_resize", Pdl::On,
                  vec ? image_resize_kernel<Src, Entry, true> : image_resize_kernel<Src, Entry, false>, grid,
                  kResizeThreads, 0, stream, dim3(1), src, tab, out, d->out_h, d->out_w, runs, total);
}

// ---------------------------------------------------------------------------------------------- Pillow filters
// Pillow's 8-bit BILINEAR and BICUBIC resamplers (include/b200_saber.h has the arithmetic). Three launches per request:
// pil_coeffs_kernel writes each image's bounds and int32 taps for its cropped output rows and columns into the
// workspace, pil_first_pass_kernel resamples the source along the image's first axis into a uint8 intermediate, and
// pil_second_pass_kernel resamples that along the other axis into `out`. Every launch depends only on the
// descriptor; the sizes, and so the tap counts, come from the device table.
constexpr int kPilPrecision = 22;
constexpr int kCoefThreads = 128;

// The workspace of one (desc, max_h, max_w, resize_short): tap records of n * (out_h + out_w) coordinates, each
// {xmin, xmax, k[kmax]} int32, then one intermediate of tmp_bytes per image.
struct PilLayout {
    int kmax, stride;                // taps per record, record size in int32
    size_t coef_bytes, tmp_bytes;
    int tmp_runs;                    // 4-pixel runs of the largest intermediate
};

// The filter's support at scale 1: 1 for the triangle (BILINEAR), 2 for the cubic (BICUBIC).
constexpr int pil_support(int filter) { return filter == B200_IMAGE_RESIZE_PIL_BICUBIC ? 2 : 1; }

// Taps are at most 2 * ceil(support) + 1 with support = f * max(in / out, 1) for the filter's support f; in <= max_*
// and the resized side is at least resize_short (S > 0) or exactly the input's side (S == 0). The horizontal-first
// intermediate is at most max_h rows of out_w pixels, the vertical-first one out_h rows of at most max_w; rows are
// padded to 4 pixels.
bool pil_layout(const b200_image_resize_desc_t* d, int filter, int max_h, int max_w, int resize_short, PilLayout* L) {
    if (filter != B200_IMAGE_RESIZE_PIL && filter != B200_IMAGE_RESIZE_PIL_BICUBIC) return false;
    if (!d || d->n < 1 || d->c < 1 || d->c > 4 || d->out_h < 1 || d->out_w < 1) return false;
    if (max_h < 1 || max_w < 1 || max_h > kMaxResized || max_w > kMaxResized || resize_short < 0) return false;
    if (resize_short != 0 && resize_short < (d->out_h > d->out_w ? d->out_h : d->out_w)) return false;
    const long long f = pil_support(filter);
    const long long min_rh = resize_short ? resize_short : d->out_h, min_rw = resize_short ? resize_short : d->out_w;
    const long long sv = (f * max_h + min_rh - 1) / min_rh, sh = (f * max_w + min_rw - 1) / min_rw;
    const long long s = sv > sh ? sv : sh;
    L->kmax = static_cast<int>(2 * (s > f ? s : f) + 1);
    L->stride = 2 + L->kmax;
    const size_t pad4_w = (d->out_w + 3) / 4 * 4, pad4_max_w = (static_cast<size_t>(max_w) + 3) / 4 * 4;
    const size_t hfirst = static_cast<size_t>(max_h) * pad4_w, vfirst = static_cast<size_t>(d->out_h) * pad4_max_w;
    const size_t tmp_px = hfirst > vfirst ? hfirst : vfirst;
    L->tmp_runs = static_cast<int>(tmp_px / 4);
    L->coef_bytes = (static_cast<size_t>(d->n) * (d->out_h + d->out_w) * L->stride * 4 + 255) / 256 * 256;
    L->tmp_bytes = (tmp_px * d->c + 255) / 256 * 256;
    return true;
}

// Pillow's Image.resize runs the vertical pass first (as a resize of its own) for an image more than 100 times taller
// than wide that shrinks in height; all other images go horizontal pass first.
__device__ __forceinline__ bool pil_vertical_first(const b200_image_resize_entry_t& e) {
    return e.h > 100ll * e.w && e.rh < e.h;
}

__device__ __forceinline__ double pil_tri(double x) {
    x = fabs(x);
    return x < 1.0 ? __dsub_rn(1.0, x) : 0.0;
}

// Pillow's bicubic_filter, a = -0.5, in Pillow's order of operations: ((a + 2) x - (a + 3)) x x + 1 on [0, 1),
// (((x - 5) x + 8) x - 4) a on [1, 2).
__device__ __forceinline__ double pil_cubic(double x) {
    x = fabs(x);
    if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
    if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
    return 0.0;
}

template <int Filter>
__device__ __forceinline__ double pil_filter(double x) {
    if constexpr (Filter == B200_IMAGE_RESIZE_PIL_BICUBIC) return pil_cubic(x);
    else return pil_tri(x);
}

// One thread = one cropped output coordinate of one image: records [img][0, out_h) are rows (o = y + top of rh, taps
// over h), [img][out_h, out_h + out_w) columns (o = x + left of rw, taps over w). Pillow's precompute_coeffs and
// normalize_coeffs_8bpc with the filter's function, every double step rounded on its own; the weights are recomputed
// for the normalisation rather than kept, which gives the same values.
template <int Filter, class Entry>
__global__ void __launch_bounds__(kCoefThreads) pil_coeffs_kernel(const Entry* __restrict__ table,
                                                                  int32_t* __restrict__ coef, int out_h, int out_w,
                                                                  int stride, long long total) {
    pdl_enter();      // the previous request's passes are done reading the records
    const long long t = blockIdx.x * 1ll * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int img = static_cast<int>(t / (out_h + out_w));
    const int j = static_cast<int>(t % (out_h + out_w));
    const bool row = j < out_h;
    const b200_image_resize_entry_t* e = resize_entry(table, img);
    const int in = row ? __ldg(&e->h) : __ldg(&e->w);
    const int out = row ? __ldg(&e->rh) : __ldg(&e->rw);
    const int o = row ? j + __ldg(&e->top) : j - out_h + __ldg(&e->left);

    const double scale = __ddiv_rn(static_cast<double>(in), static_cast<double>(out));
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    // the filter's support times the filter scale (exact: a product by 1 or 2); the taps read x / filterscale
    const double support = pil_support(Filter) == 1 ? filterscale : __dmul_rn(2.0, filterscale);
    const double ss = __ddiv_rn(1.0, filterscale);
    const double center = __dmul_rn(__dadd_rn(static_cast<double>(o), 0.5), scale);
    int xmin = __double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5));
    xmin = xmin < 0 ? 0 : xmin;
    int xmax = __double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5));
    xmax = (xmax > in ? in : xmax) - xmin;
    if (xmax > stride - 2) xmax = stride - 2;   // only for a table outside the workspace's max_h / max_w
    int32_t* rec = coef + t * stride;
    double ww = 0.0;
    for (int k = 0; k < xmax; ++k) {
        const double x = __dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(k + xmin), center), 0.5), ss);
        ww = __dadd_rn(ww, pil_filter<Filter>(x));
    }
    for (int k = 0; k < xmax; ++k) {
        double w = pil_filter<Filter>(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(k + xmin), center), 0.5), ss));
        if (ww != 0.0) w = __ddiv_rn(w, ww);
        const double v = __dmul_rn(w, static_cast<double>(1 << kPilPrecision));
        rec[2 + k] = __double2int_rz(v < 0.0 ? __dsub_rn(v, 0.5) : __dadd_rn(v, 0.5));
    }
    rec[0] = xmin;
    rec[1] = xmax;
}

// acc[ch] = 2^21 + sum_k p[k * step + ch] * taps[k] over the record's xmax taps, then clamp(acc >> 22, 0, 255).
template <int C>
__device__ __forceinline__ void pil_taps(const uint8_t* __restrict__ p, long long step,
                                         const int32_t* __restrict__ rec, uint32_t v[C]) {
    int acc[C];
#pragma unroll
    for (int ch = 0; ch < C; ++ch) acc[ch] = 1 << (kPilPrecision - 1);
    const int n = __ldg(rec + 1);
    for (int k = 0; k < n; ++k, p += step) {
        const int tap = __ldg(rec + 2 + k);
#pragma unroll
        for (int ch = 0; ch < C; ++ch) acc[ch] += static_cast<int>(__ldg(p + ch)) * tap;
    }
#pragma unroll
    for (int ch = 0; ch < C; ++ch) {
        const int r = acc[ch] >> kPilPrecision;
        v[ch] = static_cast<uint32_t>(r < 0 ? 0 : (r > 255 ? 255 : r));
    }
}

// Where the first pass's intermediate sits in the image: horizontal first, source rows [first, first + rows) of the
// out_w cropped columns; vertical first, the out_h cropped rows of source columns [first, first + cols). Rows of the
// intermediate are `pitch` pixels (cols padded to 4).
struct PilTmp {
    bool vfirst;
    int first, rows, cols, pitch;
};
template <class Entry>
__device__ __forceinline__ PilTmp pil_tmp(const Entry* table, const int32_t* coef, int img, int out_h, int out_w,
                                          int stride) {
    PilTmp m;
    const b200_image_resize_entry_t* e = resize_entry(table, img);
    b200_image_resize_entry_t ent;
    ent.h = __ldg(&e->h); ent.w = __ldg(&e->w); ent.rh = __ldg(&e->rh);
    m.vfirst = pil_vertical_first(ent);
    const int32_t* recs = coef + static_cast<long long>(img) * (out_h + out_w) * stride;
    const int32_t* lo = recs + (m.vfirst ? out_h : 0) * stride;                         // first coordinate
    const int32_t* hi = recs + (m.vfirst ? out_h + out_w - 1 : out_h - 1) * stride;     // last coordinate
    m.first = __ldg(lo);
    const int span = __ldg(hi) + __ldg(hi + 1) - m.first;
    m.rows = m.vfirst ? out_h : span;
    m.cols = m.vfirst ? span : out_w;
    m.pitch = (m.cols + 3) & ~3;
    return m;
}

// The first pass's taps of intermediate pixel (r, col) in a source layout: vertical first, the record's rows of source
// column first + col; else its columns of source row first + r.
template <int C>
__device__ __forceinline__ void pil_first_taps(const Interleaved<C>& s, const PilTmp& m, const int32_t* __restrict__ rec,
                                               int r, int col, uint32_t v[C]) {
    const long long at = m.vfirst ? static_cast<long long>(__ldg(rec)) * s.w + m.first + col
                                  : static_cast<long long>(m.first + r) * s.w + __ldg(rec);
    pil_taps<C>(s.img + at * C, m.vfirst ? 1ll * s.w * C : C, rec, v);
}
template <int F>
__device__ __forceinline__ void pil_first_taps(const Yuv420<F>& s, const PilTmp& m, const int32_t* __restrict__ rec,
                                               int r, int col, uint32_t v[3]) {
    const int y = m.vfirst ? __ldg(rec) : m.first + r, x = m.vfirst ? m.first + col : __ldg(rec);
    int acc[3];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) acc[ch] = 1 << (kPilPrecision - 1);
    const int n = __ldg(rec + 1);
    typename Yuv420<F>::Row row = s.row(y);
    for (int k = 0; k < n; ++k) {
        const int tap = __ldg(rec + 2 + k);
        if (m.vfirst) row = s.row(y + k);
        const auto p = s.pixel(row, m.vfirst ? x : x + k);
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) acc[ch] += s.tap(p, ch) * tap;
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const int q = acc[ch] >> kPilPrecision;
        v[ch] = static_cast<uint32_t>(q < 0 ? 0 : (q > 255 ? 255 : q));
    }
}

template <int C>
__device__ __forceinline__ void pil_store_run(uint8_t* o, const uint32_t (&words)[C]) {
    if constexpr (C == 4) *reinterpret_cast<uint4*>(o) = make_uint4(words[0], words[1], words[2], words[3]);
    else if constexpr (C == 2) *reinterpret_cast<uint2*>(o) = make_uint2(words[0], words[1]);
    else if constexpr (C == 3) {
        uint32_t* o32 = reinterpret_cast<uint32_t*>(o);
        o32[0] = words[0]; o32[1] = words[1]; o32[2] = words[2];
    } else *reinterpret_cast<uint32_t*>(o) = words[0];
}

// First pass. Grid (blocks, n): the blocks of one image stride over its intermediate in runs of 4 pixels of one row
// (pixels past cols are written as 0), stored as C aligned 32-bit words.
template <class Src, class Entry>
__global__ void __launch_bounds__(kResizeThreads) pil_first_pass_kernel(const uint8_t* __restrict__ src,
                                                                        const Entry* __restrict__ table,
                                                                        const int32_t* __restrict__ coef,
                                                                        uint8_t* __restrict__ tmp, size_t tmp_bytes,
                                                                        int out_h, int out_w, int stride) {
    constexpr int C = Src::kChannels;
    pdl_enter();      // the records are written; the previous request's second pass is done with tmp
    const int img = blockIdx.y;
    const PilTmp m = pil_tmp(table, coef, img, out_h, out_w, stride);
    const Src s = Src::at(src, table, img);
    const int32_t* recs = coef + static_cast<long long>(img) * (out_h + out_w) * stride;
    uint8_t* t_img = tmp + img * tmp_bytes;
    const int runs = m.pitch / 4;
    const long long total = 1ll * m.rows * runs;
    for (long long i = blockIdx.x * 1ll * blockDim.x + threadIdx.x; i < total; i += 1ll * gridDim.x * blockDim.x) {
        const int r = static_cast<int>(i / runs), x0 = static_cast<int>(i % runs) * 4;
        uint32_t words[C];
#pragma unroll
        for (int k = 0; k < C; ++k) words[k] = 0;
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int col = x0 + p;
            if (col >= m.cols) break;
            // vertical first: source column first + col, taps over rows; else source row first + r, taps over columns
            const int32_t* rec = recs + (m.vfirst ? r : out_h + col) * stride;
            uint32_t v[C];
            pil_first_taps(s, m, rec, r, col, v);
#pragma unroll
            for (int ch = 0; ch < C; ++ch) {
                const int byte = p * C + ch;
                words[byte >> 2] |= v[ch] << (8 * (byte & 3));
            }
        }
        pil_store_run<C>(t_img + (static_cast<long long>(r) * m.pitch + x0) * C, words);
    }
}

// Second pass: thread = 4 consecutive output pixels of one row, as image_resize_kernel (VEC: out_w % 4 == 0).
template <int C, class Entry, bool VEC>
__global__ void __launch_bounds__(kResizeThreads) pil_second_pass_kernel(const Entry* __restrict__ table,
                                                                         const int32_t* __restrict__ coef,
                                                                         const uint8_t* __restrict__ tmp, size_t tmp_bytes,
                                                                         uint8_t* __restrict__ out, int out_h, int out_w,
                                                                         int stride, int runs, long long total) {
    pdl_enter();      // the first pass is done; the previous request's readers of `out` are done
    const long long t = blockIdx.x * 1ll * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int run = static_cast<int>(t % runs);
    const long long row = t / runs;
    const int y = static_cast<int>(row % out_h);
    const int img = static_cast<int>(row / out_h);
    const PilTmp m = pil_tmp(table, coef, img, out_h, out_w, stride);
    const int32_t* recs = coef + static_cast<long long>(img) * (out_h + out_w) * stride;
    const uint8_t* t_img = tmp + img * tmp_bytes;
    const int x_begin = run * kPixelsPerThread;
    uint8_t* o = out + ((static_cast<long long>(img) * out_h + y) * out_w + x_begin) * C;

    uint32_t words[C];
#pragma unroll
    for (int i = 0; i < C; ++i) words[i] = 0;
#pragma unroll
    for (int p = 0; p < kPixelsPerThread; ++p) {
        const int x = x_begin + p;
        if (!VEC && x >= out_w) break;
        // vertical first: taps over the intermediate's columns; else over its rows
        const int32_t* rec = recs + (m.vfirst ? out_h + x : y) * stride;
        const long long at = m.vfirst ? static_cast<long long>(y) * m.pitch + __ldg(rec) - m.first
                                      : static_cast<long long>(__ldg(rec) - m.first) * m.pitch + x;
        uint32_t v[C];
        pil_taps<C>(t_img + at * C, m.vfirst ? C : 1ll * m.pitch * C, rec, v);
#pragma unroll
        for (int ch = 0; ch < C; ++ch) {
            if constexpr (VEC) {
                const int byte = p * C + ch;
                words[byte >> 2] |= v[ch] << (8 * (byte & 3));
            } else {
                o[p * C + ch] = static_cast<uint8_t>(v[ch]);
            }
        }
    }
    if constexpr (VEC) pil_store_run<C>(o, words);
}

template <class Src, class Entry = b200_image_resize_entry_t, int Filter = B200_IMAGE_RESIZE_PIL>
int launch_pil(const b200_image_resize_desc_t* d, const PilLayout& L, const uint8_t* src, const void* table,
               void* workspace, uint8_t* out, void* stream) {
    constexpr int C = Src::kChannels;
    const auto* tab = static_cast<const Entry*>(table);
    auto* coef = static_cast<int32_t*>(workspace);
    auto* tmp = static_cast<uint8_t*>(workspace) + L.coef_bytes;
    const long long coords = 1ll * d->n * (d->out_h + d->out_w);
    int st = launch("image_resize_pil", Pdl::On, pil_coeffs_kernel<Filter, Entry>, div_up(coords, kCoefThreads), kCoefThreads, 0, stream,
                    dim3(1), tab, coef, d->out_h, d->out_w, L.stride, coords);
    if (st != B200_SUCCESS) return st;
    // about one resident wave of threads over the batch, each image's blocks striding over its intermediate
    const long long want = 8ll * sm_count() / d->n;
    const long long need = div_up(L.tmp_runs, kResizeThreads);
    const unsigned bx = static_cast<unsigned>(want < 1 ? 1 : (want < need ? want : need));
    st = launch("image_resize_pil", Pdl::On, pil_first_pass_kernel<Src, Entry>, dim3(bx, d->n), kResizeThreads, 0, stream, dim3(1),
                src, tab, static_cast<const int32_t*>(coef), tmp, L.tmp_bytes, d->out_h, d->out_w, L.stride);
    if (st != B200_SUCCESS) return st;
    const int runs = (d->out_w + kPixelsPerThread - 1) / kPixelsPerThread;
    const long long total = 1ll * d->n * d->out_h * runs;
    const bool vec = d->out_w % kPixelsPerThread == 0;
    return launch("image_resize_pil", Pdl::On,
                  vec ? pil_second_pass_kernel<C, Entry, true> : pil_second_pass_kernel<C, Entry, false>,
                  div_up(total, kResizeThreads), kResizeThreads, 0, stream, dim3(1), tab, static_cast<const int32_t*>(coef),
                  static_cast<const uint8_t*>(tmp), L.tmp_bytes, out, d->out_h, d->out_w, L.stride, runs, total);
}

// ---------------------------------------------------------------------------------------------- OpenCV's INTER_LINEAR
// cv2.resize(img, (rw, rh)) with the default INTER_LINEAR on 8-bit images (include/b200_saber.h has the arithmetic).
// Every output pixel reads 2 x 2 taps with weights of its own row and column, so one launch does it all, with no
// workspace: each thread computes its coefficients as OpenCV's resize setup does, then sums the taps in OpenCV's
// fixed point.
constexpr int kCv2CoefScale = 1 << 11;      // INTER_RESIZE_COEF_SCALE

struct Cv2Axis {
    int s0, s1;     // source taps
    int a0, a1;     // their 11-bit weights
};

// Output coordinate d of a side resized in -> out, scale = 1.0 / ((double)out / in), in double and fp32 with every
// step rounded on its own. Columns clamp both taps and the fraction at the edges; rows clamp only the taps, as
// OpenCV's vertical pass reads the weights of the unclamped fraction.
template <bool Columns>
__device__ __forceinline__ Cv2Axis cv2_axis(double scale, int d, int in) {
    float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn(static_cast<double>(d), 0.5), scale), 0.5));
    int s = __float2int_rd(f);
    f = __fsub_rn(f, static_cast<float>(s));
    Cv2Axis a;
    if (Columns) {
        if (s < 0) s = 0, f = 0.f;
        if (s + 1 >= in) s = in - 1, f = 0.f;
        a.s0 = s;
        a.s1 = f == 0.f ? s : s + 1;      // a1 is 0 when f is
    } else {
        a.s0 = s < 0 ? 0 : (s > in - 1 ? in - 1 : s);
        a.s1 = s + 1 < 0 ? 0 : (s + 1 > in - 1 ? in - 1 : s + 1);
    }
    a.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), static_cast<float>(kCv2CoefScale)));
    a.a1 = __float2int_rn(__fmul_rn(f, static_cast<float>(kCv2CoefScale)));
    return a;
}

__device__ __forceinline__ double cv2_scale(int in, int out) {
    return __ddiv_rn(1.0, __ddiv_rn(static_cast<double>(out), static_cast<double>(in)));
}

// Thread = kPixelsPerThread consecutive output pixels of one row of one image, as image_resize_kernel (VEC:
// out_w % 4 == 0). The sum of the two weighted rows is at most 1020, so the result needs no clamp.
template <class Src, class Entry, bool VEC>
__global__ void __launch_bounds__(kResizeThreads) cv2_linear_kernel(const uint8_t* __restrict__ src,
                                                                    const Entry* __restrict__ table,
                                                                    uint8_t* __restrict__ out, int out_h, int out_w,
                                                                    int runs, long long total) {
    constexpr int C = Src::kChannels;
    pdl_enter();      // the previous request's readers of `out` are done
    const long long t = blockIdx.x * 1ll * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int run = static_cast<int>(t % runs);
    const long long row = t / runs;
    const int y = static_cast<int>(row % out_h);
    const int img = static_cast<int>(row / out_h);
    const b200_image_resize_entry_t* e = resize_entry(table, img);
    const long long offset = __ldg(&e->offset);
    const int h = __ldg(&e->h), w = __ldg(&e->w);
    const int rh = __ldg(&e->rh), rw = __ldg(&e->rw);
    const int top = __ldg(&e->top), left = __ldg(&e->left);
    // OpenCV resizes a two-channel image shrunk exactly 2x on both axes with its float area filter, whose sum of the
    // 2 x 2 block rounds half to even; every other 2x shrink gives (sum + 2) >> 2, which the sums below equal.
    const bool area_half_even = C == 2 && h == 2 * rh && w == 2 * rw;

    const Cv2Axis ay = cv2_axis<false>(cv2_scale(h, rh), y + top, h);
    const Src s(src + offset, box_of(table + img, h, w));
    const auto r0 = s.row(ay.s0);
    const auto r1 = s.row(ay.s1);
    const double sx = cv2_scale(w, rw);
    const int x_begin = run * kPixelsPerThread;
    uint8_t* o = out + ((static_cast<long long>(img) * out_h + y) * out_w + x_begin) * C;

    uint32_t words[C];
#pragma unroll
    for (int i = 0; i < C; ++i) words[i] = 0;
#pragma unroll
    for (int p = 0; p < kPixelsPerThread; ++p) {
        if (!VEC && x_begin + p >= out_w) break;
        const Cv2Axis ax = cv2_axis<true>(sx, x_begin + p + left, w);
        const auto q00 = s.pixel(r0, ax.s0), q01 = s.pixel(r0, ax.s1);
        const auto q10 = s.pixel(r1, ax.s0), q11 = s.pixel(r1, ax.s1);
#pragma unroll
        for (int ch = 0; ch < C; ++ch) {
            // the horizontal sums are exact in int32; the vertical one drops 4 bits, then 16, then rounds off 2
            const int s0 = static_cast<int>(s.tap(q00, ch)) * ax.a0 + static_cast<int>(s.tap(q01, ch)) * ax.a1;
            const int s1 = static_cast<int>(s.tap(q10, ch)) * ax.a0 + static_cast<int>(s.tap(q11, ch)) * ax.a1;
            const int v = (((s0 >> 4) * ay.a0) >> 16) + (((s1 >> 4) * ay.a1) >> 16);
            const uint32_t b = static_cast<uint32_t>((v + (area_half_even ? 1 + ((v >> 2) & 1) : 2)) >> 2);
            if constexpr (VEC) {
                const int byte = p * C + ch;
                words[byte >> 2] |= b << (8 * (byte & 3));
            } else {
                o[p * C + ch] = static_cast<uint8_t>(b);
            }
        }
    }
    if constexpr (VEC) pil_store_run<C>(o, words);
}

template <class Src, class Entry>
int launch_cv2_linear(const b200_image_resize_desc_t* d, const uint8_t* src, const void* table, uint8_t* out,
                      void* stream) {
    const int runs = (d->out_w + kPixelsPerThread - 1) / kPixelsPerThread;
    const long long total = 1ll * d->n * d->out_h * runs;
    const auto* tab = static_cast<const Entry*>(table);
    const bool vec = d->out_w % kPixelsPerThread == 0;
    return launch("image_resize_cv2_linear", Pdl::On,
                  vec ? cv2_linear_kernel<Src, Entry, true> : cv2_linear_kernel<Src, Entry, false>,
                  div_up(total, kResizeThreads), kResizeThreads, 0, stream, dim3(1), src, tab, out, d->out_h,
                  d->out_w, runs, total);
}

// Any filter on a table of b200_image_crop_entry_t
template <class Src>
int launch_crop(const b200_image_resize_desc_t* d, int filter, const PilLayout& L, const uint8_t* src,
                const void* table, void* workspace, uint8_t* out, void* stream) {
    using Crop = b200_image_crop_entry_t;
    if (filter == B200_IMAGE_RESIZE_CV2_LINEAR) return launch_cv2_linear<Src, Crop>(d, src, table, out, stream);
    if (filter == B200_IMAGE_RESIZE_PIL)
        return launch_pil<Src, Crop, B200_IMAGE_RESIZE_PIL>(d, L, src, table, workspace, out, stream);
    if (filter == B200_IMAGE_RESIZE_PIL_BICUBIC)
        return launch_pil<Src, Crop, B200_IMAGE_RESIZE_PIL_BICUBIC>(d, L, src, table, workspace, out, stream);
    return launch_resize<Src, Crop>(d, src, table, out, stream);
}

}  // namespace
}  // namespace b200

extern "C" {

int b200_image_resize_geometry(int32_t h, int32_t w, int32_t resize_short, int32_t out_h, int32_t out_w, int32_t* rh,
                               int32_t* rw, int32_t* top, int32_t* left) {
    using b200::kMaxResized;
    if (!rh || !rw || !top || !left) return B200_INVALID_VALUE;
    if (h < 1 || w < 1 || out_h < 1 || out_w < 1 || h > kMaxResized || w > kMaxResized || resize_short < 0)
        return B200_INVALID_VALUE;
    long long sh, sw;
    if (resize_short == 0) {
        sh = out_h;
        sw = out_w;
    } else {
        if (resize_short < (out_h > out_w ? out_h : out_w)) return B200_INVALID_VALUE;
        const long long s = resize_short;
        if (h <= w) { sh = s; sw = s * w / h; }
        else { sw = s; sh = s * h / w; }
    }
    if (sh > kMaxResized || sw > kMaxResized) return B200_INVALID_VALUE;
    *rh = static_cast<int32_t>(sh);
    *rw = static_cast<int32_t>(sw);
    *top = static_cast<int32_t>((sh - out_h) / 2);
    *left = static_cast<int32_t>((sw - out_w) / 2);
    return B200_SUCCESS;
}

int b200_image_resize_run(const b200_image_resize_desc_t* d, const uint8_t* src, const void* table_dev, uint8_t* out,
                          void* stream) {
    if (!d || !src || !table_dev || !out) return B200_INVALID_VALUE;
    if (d->n < 1 || d->c < 1 || d->c > 4 || d->out_h < 1 || d->out_w < 1) return B200_INVALID_VALUE;
    if (!b200::device_is_sm90()) return B200_WRONG_DEVICE;
    switch (d->c) {
        case 1: return b200::launch_resize<b200::Interleaved<1>>(d, src, table_dev, out, stream);
        case 2: return b200::launch_resize<b200::Interleaved<2>>(d, src, table_dev, out, stream);
        case 3: return b200::launch_resize<b200::Interleaved<3>>(d, src, table_dev, out, stream);
        default: return b200::launch_resize<b200::Interleaved<4>>(d, src, table_dev, out, stream);
    }
}

int b200_image_resize_geometry_ex(int32_t h, int32_t w, int32_t resize_short, int32_t out_h, int32_t out_w,
                                  int32_t filter, int32_t* rh, int32_t* rw, int32_t* top, int32_t* left) {
    if (filter != B200_IMAGE_RESIZE_REFERENCE && filter != B200_IMAGE_RESIZE_PIL &&
        filter != B200_IMAGE_RESIZE_PIL_BICUBIC && filter != B200_IMAGE_RESIZE_CV2_LINEAR)
        return B200_INVALID_VALUE;
    const int st = b200_image_resize_geometry(h, w, resize_short, out_h, out_w, rh, rw, top, left);
    // the floor offsets of an OpenCV caller's img[(rh - H) // 2:..., (rw - W) // 2:...]
    if (st != B200_SUCCESS || filter == B200_IMAGE_RESIZE_REFERENCE || filter == B200_IMAGE_RESIZE_CV2_LINEAR)
        return st;
    // torchvision CenterCrop: round((r - out) / 2.0), half to even
    const int32_t dh = *rh - out_h, dw = *rw - out_w;
    *top = dh / 2 + ((dh & 1) & ((dh / 2) & 1));
    *left = dw / 2 + ((dw & 1) & ((dw / 2) & 1));
    return B200_SUCCESS;
}

int b200_image_resize_workspace(const b200_image_resize_desc_t* d, int32_t filter, int32_t max_h, int32_t max_w,
                                int32_t resize_short, size_t* bytes) {
    if (!bytes || !d) return B200_INVALID_VALUE;
    if (filter == B200_IMAGE_RESIZE_REFERENCE || filter == B200_IMAGE_RESIZE_CV2_LINEAR) {
        if (d->n < 1 || d->c < 1 || d->c > 4 || d->out_h < 1 || d->out_w < 1) return B200_INVALID_VALUE;
        *bytes = 0;
        return B200_SUCCESS;
    }
    b200::PilLayout L;
    if (!b200::pil_layout(d, filter, max_h, max_w, resize_short, &L)) return B200_INVALID_VALUE;
    *bytes = L.coef_bytes + static_cast<size_t>(d->n) * L.tmp_bytes;
    return B200_SUCCESS;
}

int b200_image_resize_pil_workspace(const b200_image_resize_desc_t* d, int32_t max_h, int32_t max_w,
                                    int32_t resize_short, size_t* bytes) {
    return b200_image_resize_workspace(d, B200_IMAGE_RESIZE_PIL, max_h, max_w, resize_short, bytes);
}

int b200_image_resize_pil_run(const b200_image_resize_desc_t* d, int32_t max_h, int32_t max_w, int32_t resize_short,
                              const uint8_t* src, const void* table_dev, void* workspace, uint8_t* out, void* stream) {
    b200::PilLayout L;
    if (!src || !table_dev || !workspace || !out ||
        !b200::pil_layout(d, B200_IMAGE_RESIZE_PIL, max_h, max_w, resize_short, &L))
        return B200_INVALID_VALUE;
    if (!b200::device_is_sm90()) return B200_WRONG_DEVICE;
    switch (d->c) {
        case 1: return b200::launch_pil<b200::Interleaved<1>>(d, L, src, table_dev, workspace, out, stream);
        case 2: return b200::launch_pil<b200::Interleaved<2>>(d, L, src, table_dev, workspace, out, stream);
        case 3: return b200::launch_pil<b200::Interleaved<3>>(d, L, src, table_dev, workspace, out, stream);
        default: return b200::launch_pil<b200::Interleaved<4>>(d, L, src, table_dev, workspace, out, stream);
    }
}

int b200_image_resize_yuv_run(const b200_image_resize_desc_t* d, int32_t format, const uint8_t* src,
                              const void* table_dev, uint8_t* out, void* stream) {
    if (!d || d->c != 3 || (format != B200_IMAGE_YUV_NV12 && format != B200_IMAGE_YUV_I420)) return B200_INVALID_VALUE;
    if (!src || !table_dev || !out || d->n < 1 || d->out_h < 1 || d->out_w < 1) return B200_INVALID_VALUE;
    if (!b200::device_is_sm90()) return B200_WRONG_DEVICE;
    if (format == B200_IMAGE_YUV_NV12)
        return b200::launch_resize<b200::Yuv420<B200_IMAGE_YUV_NV12>>(d, src, table_dev, out, stream);
    return b200::launch_resize<b200::Yuv420<B200_IMAGE_YUV_I420>>(d, src, table_dev, out, stream);
}

int b200_image_resize_pil_yuv_run(const b200_image_resize_desc_t* d, int32_t format, int32_t max_h, int32_t max_w,
                                  int32_t resize_short, const uint8_t* src, const void* table_dev, void* workspace,
                                  uint8_t* out, void* stream) {
    b200::PilLayout L;
    if (!d || d->c != 3 || (format != B200_IMAGE_YUV_NV12 && format != B200_IMAGE_YUV_I420)) return B200_INVALID_VALUE;
    if (!src || !table_dev || !workspace || !out ||
        !b200::pil_layout(d, B200_IMAGE_RESIZE_PIL, max_h, max_w, resize_short, &L))
        return B200_INVALID_VALUE;
    if (!b200::device_is_sm90()) return B200_WRONG_DEVICE;
    if (format == B200_IMAGE_YUV_NV12)
        return b200::launch_pil<b200::Yuv420<B200_IMAGE_YUV_NV12>>(d, L, src, table_dev, workspace, out, stream);
    return b200::launch_pil<b200::Yuv420<B200_IMAGE_YUV_I420>>(d, L, src, table_dev, workspace, out, stream);
}

int b200_image_crop_resize_run(const b200_image_resize_desc_t* d, int32_t filter, int32_t pixel_format, int32_t max_h,
                               int32_t max_w, int32_t resize_short, const uint8_t* src, const void* table_dev,
                               void* workspace, uint8_t* out, void* stream) {
    const bool pil = filter == B200_IMAGE_RESIZE_PIL || filter == B200_IMAGE_RESIZE_PIL_BICUBIC;
    if (!d || (!pil && filter != B200_IMAGE_RESIZE_REFERENCE && filter != B200_IMAGE_RESIZE_CV2_LINEAR))
        return B200_INVALID_VALUE;
    if (pixel_format != B200_IMAGE_INTERLEAVED && pixel_format != B200_IMAGE_YUV_NV12 &&
        pixel_format != B200_IMAGE_YUV_I420)
        return B200_INVALID_VALUE;
    if (pixel_format != B200_IMAGE_INTERLEAVED && d->c != 3) return B200_INVALID_VALUE;
    if (!src || !table_dev || !out || (pil && !workspace)) return B200_INVALID_VALUE;
    if (d->n < 1 || d->c < 1 || d->c > 4 || d->out_h < 1 || d->out_w < 1) return B200_INVALID_VALUE;
    b200::PilLayout L;
    if (pil && !b200::pil_layout(d, filter, max_h, max_w, resize_short, &L)) return B200_INVALID_VALUE;
    if (!b200::device_is_sm90()) return B200_WRONG_DEVICE;
    if (pixel_format == B200_IMAGE_YUV_NV12)
        return b200::launch_crop<b200::Yuv420<B200_IMAGE_YUV_NV12>>(d, filter, L, src, table_dev, workspace, out, stream);
    if (pixel_format == B200_IMAGE_YUV_I420)
        return b200::launch_crop<b200::Yuv420<B200_IMAGE_YUV_I420>>(d, filter, L, src, table_dev, workspace, out, stream);
    switch (d->c) {
        case 1: return b200::launch_crop<b200::Interleaved<1>>(d, filter, L, src, table_dev, workspace, out, stream);
        case 2: return b200::launch_crop<b200::Interleaved<2>>(d, filter, L, src, table_dev, workspace, out, stream);
        case 3: return b200::launch_crop<b200::Interleaved<3>>(d, filter, L, src, table_dev, workspace, out, stream);
        default: return b200::launch_crop<b200::Interleaved<4>>(d, filter, L, src, table_dev, workspace, out, stream);
    }
}

}  // extern "C"
