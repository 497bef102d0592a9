// common.cuh -- shared helpers for libb200_roi_ops.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../../include/b200_roi_ops.h"

namespace b200 {

// ---- launch accounting / error plumbing -------------------------------------------------------
extern unsigned long long g_launch_count;   // defined in api.cu

inline int finish_launch(int n_launches = 1) {
    __atomic_fetch_add(&g_launch_count, (unsigned long long)n_launches, __ATOMIC_RELAXED);   // callers may be one thread per GPU
    cudaError_t err = cudaGetLastError();
    return (err == cudaSuccess) ? B200_ROI_OK : (int)err;
}

constexpr int kNumSMs = 132;   // H100 SXM

// ---- per-device kernel setup (api.cu) -------------------------------------------------------------
// Makes `kernel` launchable with `bytes` of dynamic shared memory on the current device.  The limit only ever rises: it is
// set under one lock, the first time a (kernel, device) pair needs more than the limit already recorded for it, so calls
// from several host threads never lower a limit another call is about to launch with.  Requests of 48 KB or less return at
// once.  On failure, clears the CUDA error and returns it; the caller decides whether that means decline or error.
int smem_opt_in(const void* kernel, size_t bytes);
template <class K> int smem_opt_in(K* kernel, size_t bytes) { return smem_opt_in((const void*)kernel, bytes); }

// SM count of the current device, queried once per device (0 / error status on failure).
int device_sm_count(int* sm_count);

// Status of a fast path that does not apply to the shape or workspace it was given: the caller falls back to another path.
// Neither B200_ROI_OK, a negative B200_ROI_E* code nor a CUDA runtime error (those stop at cudaErrorUnknown = 999).
constexpr int kPathDeclined = 1000;

// ---- dispatch switches -------------------------------------------------------------------------
// Test overrides of the path selection, which otherwise follows the shape.  Each switch is read from the environment ONCE
// (first use) and can be changed afterwards through b200_roi_ops_set_option() -- the hot path never calls getenv().
// The value is the first character of the string ('\0' = auto / default).
enum Option {
    kOptFwdPath = 0,      // B200_ROI_ALIGN_PATH      = auto | generic | tiled | stream | quad (auto: stream first, then quad; api.cu)
    kOptBwdPath,          // B200_ROI_ALIGN_BWD_PATH  = auto | generic | nhwc | rows
    kNumOptions
};
int option_get(Option which);

// ---- RoIAlign paths behind the dispatch in api.cu ----------------------------------------------------------------------------
// Defined in roi_align_<path>.cu.  row_map (nullable) gives each RoI's output row; a fast path returns kPathDeclined when the
// shape or the workspace does not suit it.
int roi_align_forward_generic(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                              const float* rois, float* top, const int* row_map, cudaStream_t stream);
int roi_align_backward_generic(const float* top_diff, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                               const float* rois, float* bottom_diff, const int* row_map, cudaStream_t stream);
size_t roi_align_tiled_workspace_bytes(int N, int R, int H, int W, int PH, int PW, int sr);
int roi_align_forward_tiled(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                            const float* rois, float* top, const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t roi_align_stream_workspace_bytes(int N, int R, int H, int W, int PH, int PW, int sr);
int roi_align_forward_stream(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                             const float* rois, float* top, const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t roi_align_strip_workspace_bytes(int N, int R, int H, int W, int PH, int PW, int sr);
int roi_align_forward_strip(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                            const float* rois, float* top, const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t roi_align_strip_fpn_workspace_bytes(int levels, const int* heights, const int* widths, int N, int R, int PH, int PW, int sr);
int roi_align_forward_strip_fpn(int levels, const float* const* bottoms, const int* heights, const int* widths, const float* scales,
                                const int* level_roi_begin, int N, int R, int C, int PH, int PW, int sr, const float* rois, float* top,
                                const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream);
size_t roi_align_bwd_nhwc_workspace_bytes(int N, int C, int H, int W);
int roi_align_backward_nhwc(const float* top_diff, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                            const float* rois, float* bottom_diff, const int* row_map, void* workspace, size_t workspace_bytes,
                            cudaStream_t stream);
size_t roi_align_bwd_rows_workspace_bytes(int N, int R, int C, int H, int W, int PH, int PW, int sr);
int roi_align_backward_rows(const float* top_diff, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                            const float* rois, float* bottom_diff, const int* row_map, void* workspace, size_t workspace_bytes,
                            cudaStream_t stream);
// Transposes a channel-innermost gradient image back to NCHW (roi_align_bwd_nhwc.cu; RoICrop's backward uses it too).
void launch_nhwc_to_nchw(const float* scratch, float* dx, int N, int C, int HW, cudaStream_t stream);

// Watchdog records of the streaming and quad-strip paths (b200_roi_ops_debug_timing_buffer).
void roi_align_stream_set_debug_buffer(unsigned long long* host_pinned);
void roi_align_strip_set_debug_buffer(unsigned long long* host_pinned);

// Dimension check shared by the RoIAlign, legacy RoIAlign and RoIPool entry points.
inline bool bad_dims(int N, int R, int H, int W, int C, int PH, int PW) {
    return N < 0 || R < 0 || H <= 0 || W <= 0 || C < 0 || PH <= 0 || PW <= 0;
}

// ---- arithmetic that must round exactly like the reference kernels' SASS --------------------
// All helpers use the _rn intrinsics, which nvcc never contracts or re-associates, so the
// fusion pattern is exactly what is written here (see oracle/roi_ops_oracle.c for the recipes
// and how they were read off `cuobjdump -sass` of the reference kernels built for sm_90a).

// RoI geometry of the Caffe2-exact RoIAlign (reference roi_align_kernel.cu:75-98).
struct XfromRoi {
    int   batch;
    float start_w, start_h, bin_w, bin_h;
    int   grid_w, grid_h;
};

__device__ __forceinline__ XfromRoi xfrom_roi(const float* __restrict__ roi, float scale, int PH, int PW, int sr) {
    XfromRoi g;
    g.batch = (int)roi[0];
    g.start_w = __fmul_rn(roi[1], scale);
    g.start_h = __fmul_rn(roi[2], scale);
    float rw = fmaxf(__fmaf_rn(roi[3], scale, -g.start_w), 1.f);
    float rh = fmaxf(__fmaf_rn(roi[4], scale, -g.start_h), 1.f);
    g.bin_h = __fdiv_rn(rh, (float)PH);
    g.bin_w = __fdiv_rn(rw, (float)PW);
    g.grid_h = (sr > 0) ? sr : (int)ceilf(g.bin_h);
    g.grid_w = (sr > 0) ? sr : (int)ceilf(g.bin_w);
    return g;
}

// sample coordinate: FADD(FFMA(p, bin, start), FMUL(i + .5, bin) / grid)   (:106-110)
__device__ __forceinline__ float xfrom_coord(float start, float bin, int p, int i, int grid) {
    float base = __fmaf_rn((float)p, bin, start);
    float off = __fdiv_rn(__fmul_rn(__fadd_rn((float)i, .5f), bin), (float)grid);
    return __fadd_rn(base, off);
}

// One axis of bilinear_interpolate (:19-52): low/high cell and the two weights (l = frac, h = 1-l).
// valid == false  <=>  the reference's "outside the map" early-out for this axis.
struct AxisTap {
    int   low, high;
    float l, h;
    bool  valid;
};

__device__ __forceinline__ AxisTap xfrom_axis(float v, int size) {
    AxisTap t;
    t.valid = !(v < -1.0f || v > (float)size);
    if (v <= 0.f) v = 0.f;
    int low = (int)v;
    if (low >= size - 1) {
        t.low = t.high = size - 1;
        v = (float)(size - 1);
    } else {
        t.low = low;
        t.high = low + 1;
    }
    t.l = __fsub_rn(v, (float)t.low);
    t.h = __fsub_rn(1.f, t.l);
    return t;
}

// ---- one axis of cv2.resize's float32 INTER_LINEAR (imgproc resize.cpp, IPP off) ----------------------------------------
// Output index d, scale = 1 / inv_scale in double: f = float((d + .5) * scale - .5), s = floor(f), f -= s.  On the x axis
// (clamp) a position before the first / past the last source column is clamped to it with f = 0; on the y axis f is kept
// and both indices s, s + 1 are clipped into [0, src).  Weights w0 = 1 - f, w1 = f.
struct Cv2Tap {
    int s0, s1;
    float w0, w1;
};

__device__ __forceinline__ Cv2Tap cv2_linear_tap(long long d, double scale, int src, bool clamp) {
    float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, .5), scale), .5));
    const float fl = floorf(f);
    int s = (int)fl;
    f = __fsub_rn(f, fl);
    if (clamp) {
        if (s < 0) { f = 0.f; s = 0; }
        if (s >= src - 1) { f = 0.f; s = src - 1; }
    }
    Cv2Tap t;
    t.s0 = s < 0 ? 0 : (s > src - 1 ? src - 1 : s);
    t.s1 = s + 1 < 0 ? 0 : (s + 1 > src - 1 ? src - 1 : s + 1);
    t.w0 = __fsub_rn(1.f, f);
    t.w1 = f;
    return t;
}

// ---- IoU exactly as the reference's compiled Cython computes it (lib/utils/cython_bbox.pyx:52-72) ----------------------
// The generated C adds the literal 1.0 as a DOUBLE: widths / heights are (double)(float difference) + 1.0, their products and the
// union are formed in double (separate multiply and add: x86-64 baseline has no FMA) and rounded to float once on assignment
// (box_area, iw, ih, ua are float variables); the final quotient (iw * ih) / ua is float.  Up to 2 ulp away from an all-float
// evaluation -- enough to flip a threshold test.
__device__ __forceinline__ float cython_area(float x1, float y1, float x2, float y2) {
    return (float)__dmul_rn(__dadd_rn((double)__fsub_rn(x2, x1), 1.0), __dadd_rn((double)__fsub_rn(y2, y1), 1.0));
}
// b: the "boxes" row, q: the "query_boxes" row, qarea = cython_area(q)
__device__ __forceinline__ float cython_iou(float bx1, float by1, float bx2, float by2, float qx1, float qy1, float qx2, float qy2,
                                            float qarea) {
    const float iw = (float)__dadd_rn((double)__fsub_rn(fminf(bx2, qx2), fmaxf(bx1, qx1)), 1.0);
    if (!(iw > 0.f)) return 0.f;
    const float ih = (float)__dadd_rn((double)__fsub_rn(fminf(by2, qy2), fmaxf(by1, qy1)), 1.0);
    if (!(ih > 0.f)) return 0.f;
    const float inter = __fmul_rn(iw, ih);
    const double barea = __dmul_rn(__dadd_rn((double)__fsub_rn(bx2, bx1), 1.0), __dadd_rn((double)__fsub_rn(by2, by1), 1.0));
    const float ua = (float)__dsub_rn(__dadd_rn(barea, (double)qarea), (double)inter);
    return __fdiv_rn(inter, ua);
}

}  // namespace b200
