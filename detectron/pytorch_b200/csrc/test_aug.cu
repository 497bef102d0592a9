// test_aug.cu -- test-time augmentation of the mask and keypoint heads (lib/core/test.py:365-729 im_detect_mask_aug /
// im_detect_keypoints_aug / combine_heatmaps_size_dep) and the width-relative aspect-ratio resize of the input image
// (lib/utils/image.py:27-32 aspect_ratio_rel).
//
// Combine: the reference stacks the T head outputs on the host and reduces them with np.mean / np.amax over axis 0.  numpy
// reduces an outer axis one slice at a time, so the result is a running fold in transform order, which is what these kernels
// do as the transforms arrive: b200_tta_combine folds one transform into acc (R, C, M, M), b200_tta_finish divides.
//   AVG (SOFT_AVG / HM_AVG):  acc = 0 + a0 (numpy's add.reduce starts from its identity, so -0.0 becomes +0.0), then acc + a_t,
//                             finally acc / n in float32.
//   MAX (SOFT_MAX / HM_MAX):  acc = a0, then np.maximum(acc, a_t) = (acc > a_t || acc is NaN) ? acc : a_t (NaN propagates, and
//                             of two equal values the later one is kept: max(-0.0, +0.0) is +0.0, max(+0.0, -0.0) is -0.0).
//   LOGIT_AVG:                AVG over -1.0 * log((1 - y) / np.maximum(y, 1e-20)) in float32, finally 1 / (1 + exp(-acc / n)).
//                             log and exp are evaluated in double and rounded once; numpy's SIMD float32 log / exp are not
//                             correctly rounded, so this mode agrees with numpy to a few ulps, not bit for bit.
// A source is read mirrored along its last axis (hflip: [..., ::-1]) and through an optional channel permutation
// (keypoint_utils.flip_heatmaps: output channel c reads source channel perm[c]); per-row ops select the first included
// transform of a row, a later one, or none (combine_heatmaps_size_dep's per-object selection).
//
// Work layout: one thread per 4 consecutive elements of a row of M (float4 loads and stores, the mirrored read a reversed
// float4) when M % 4 == 0 and the buffers are 16-byte aligned, else one thread per element.  Each call reads the source and
// acc once and writes acc once: 3 * R * C * M * M * 4 bytes, the first transform 2x.
//
// Aspect-ratio resize: cv2.resize(im, (W', h)) of a uint8 (h, w, 3) image, INTER_LINEAR with cv2's 8-bit fixed-point
// arithmetic (IPP off): per output column dx, fx = float((dx + 0.5) * (1 / (W' / w)) - 0.5), sx = floor(fx), fx -= sx, both
// borders clamped (fx = 0), alpha = (rint((1 - fx) * 2048), rint(fx * 2048)); the horizontal sum is an int and the vertical
// stage (height unchanged: weights (2048, 0)) is (((2048 * (s >> 4)) >> 16) + 2) >> 2 = (s + 1024) >> 11.  One thread per
// output pixel (3 bytes); an image is a few MB and stays in L2.
#include "common.cuh"

namespace b200 {

namespace {
constexpr int kCombineThreads = 256;
constexpr int kResizeThreads = 256;

enum Heur { kAvg = 0, kMax = 1, kLogitAvg = 2 };

__device__ __forceinline__ float np_logit(float y) {
    const float num = __fsub_rn(1.f, y);
    const float den = (y > 1e-20f || y != y) ? y : 1e-20f;              // np.maximum(y, 1e-20)
    return -(float)log((double)__fdiv_rn(num, den));
}

__device__ __forceinline__ float np_max(float a, float b) { return (a > b || a != a) ? a : b; }

__device__ __forceinline__ float fold(float acc, float v, int heur, bool first) {
    if (heur == kMax) return first ? v : np_max(acc, v);
    return __fadd_rn(first ? 0.f : acc, v);
}

// grid over (R, C, M, M / vw) element groups; vw = 4 (vectorised) or 1
template <int VW>
__global__ void __launch_bounds__(kCombineThreads)
tta_combine_kernel(const float* __restrict__ src, float* __restrict__ acc, int C, int M, long long groups, const int* __restrict__ perm,
                   const unsigned char* __restrict__ row_op, int op, bool hflip, int heur) {
    const long long g = (long long)blockIdx.x * kCombineThreads + threadIdx.x;
    if (g >= groups) return;
    const int gpr = M / VW;                                              // groups per spatial row
    const long long e = g * VW;                                          // first element of the group in (R, C, M, M)
    const long long plane = (long long)M * M;
    const long long rc = e / plane;
    const int r = (int)(rc / C), c = (int)(rc % C);
    const int y = (int)((e % plane) / M), x0 = (int)(g % gpr) * VW;
    const int o = row_op ? (int)row_op[r] : op;
    if (o == 0) return;
    const int sc = perm ? __ldg(perm + c) : c;
    const long long src_row = (((long long)r * C + sc) * M + y) * M;
    float v[VW], a[VW];
    if (VW == 4) {
        const int sx = hflip ? M - 4 - x0 : x0;
        const float4 q = __ldg(reinterpret_cast<const float4*>(src + src_row + sx));
        if (hflip) { v[0] = q.w; v[1] = q.z; v[2] = q.y; v[3] = q.x; }
        else       { v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w; }
    } else {
        v[0] = __ldg(src + src_row + (hflip ? M - 1 - x0 : x0));
    }
    const bool first = o == 1;
    if (!first) {
        if (VW == 4) {
            const float4 p = *reinterpret_cast<const float4*>(acc + e);
            a[0] = p.x; a[1] = p.y; a[2] = p.z; a[3] = p.w;
        } else {
            a[0] = acc[e];
        }
    }
#pragma unroll
    for (int j = 0; j < VW; ++j) {
        const float t = heur == kLogitAvg ? np_logit(v[j]) : v[j];
        a[j] = fold(first ? 0.f : a[j], t, heur, first);
    }
    if (VW == 4) *reinterpret_cast<float4*>(acc + e) = make_float4(a[0], a[1], a[2], a[3]);
    else acc[e] = a[0];
}

__global__ void __launch_bounds__(kCombineThreads)
tta_finish_kernel(float* __restrict__ acc, long long row_elems, long long n, const int* __restrict__ row_count, int count, int heur) {
    const long long i = (long long)blockIdx.x * kCombineThreads + threadIdx.x;
    if (i >= n) return;
    const float k = (float)(row_count ? row_count[i / row_elems] : count);
    const float m = __fdiv_rn(acc[i], k);
    acc[i] = heur == kLogitAvg ? __fdiv_rn(1.f, __fadd_rn(1.f, (float)exp(-(double)m))) : m;
}

__global__ void __launch_bounds__(kResizeThreads)
resize_width_u8_kernel(const unsigned char* __restrict__ src, long long src_pitch, int h, int w, int out_w, double scale_x,
                       unsigned char* __restrict__ dst) {
    const long long t = (long long)blockIdx.x * kResizeThreads + threadIdx.x;
    if (t >= (long long)h * out_w) return;
    const int y = (int)(t / out_w), dx = (int)(t % out_w);
    float fx = (float)((dx + 0.5) * scale_x - 0.5);
    int sx = (int)floorf(fx);
    fx -= (float)sx;
    if (sx < 0) fx = 0.f, sx = 0;
    if (sx >= w - 1) fx = 0.f, sx = w - 1;
    const int a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f));
    const int a1 = __float2int_rn(__fmul_rn(fx, 2048.f));
    const int sx1 = min(sx + 1, w - 1);
    const unsigned char* row = src + (long long)y * src_pitch;
    unsigned char* out = dst + 3 * t;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int s = (int)__ldg(row + 3 * sx + c) * a0 + (int)__ldg(row + 3 * sx1 + c) * a1;
        out[c] = (unsigned char)min(max((s + 1024) >> 11, 0), 255);
    }
}
}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_tta_combine(const float* src, float* acc, int num_rows, int num_channels, int resolution, const int* channel_perm,
                     const unsigned char* row_op, int op, int hflip, int heur, b200_stream_t stream) {
    if (!src || !acc || num_rows < 0 || num_channels < 1 || resolution < 1 || resolution > 4096) return B200_ROI_EINVAL;
    if (heur < kAvg || heur > kLogitAvg || (!row_op && op != 1 && op != 2)) return B200_ROI_EINVAL;
    const long long n = (long long)num_rows * num_channels * resolution * resolution;
    if (n == 0) return B200_ROI_OK;
    const bool vec = resolution % 4 == 0 && reinterpret_cast<uintptr_t>(src) % 16 == 0 && reinterpret_cast<uintptr_t>(acc) % 16 == 0;
    const long long groups = vec ? n / 4 : n;
    const unsigned blocks = (unsigned)((groups + kCombineThreads - 1) / kCombineThreads);
    if (vec)
        tta_combine_kernel<4><<<blocks, kCombineThreads, 0, stream>>>(src, acc, num_channels, resolution, groups, channel_perm, row_op, op,
                                                                      hflip != 0, heur);
    else
        tta_combine_kernel<1><<<blocks, kCombineThreads, 0, stream>>>(src, acc, num_channels, resolution, groups, channel_perm, row_op, op,
                                                                      hflip != 0, heur);
    return finish_launch(1);
}

int b200_tta_finish(float* acc, int num_rows, int num_channels, int resolution, const int* row_count, int count, int heur,
                    b200_stream_t stream) {
    if (!acc || num_rows < 0 || num_channels < 1 || resolution < 1 || resolution > 4096) return B200_ROI_EINVAL;
    if (heur < kAvg || heur > kLogitAvg || (!row_count && count < 1)) return B200_ROI_EINVAL;
    const long long row_elems = (long long)num_channels * resolution * resolution;
    const long long n = (long long)num_rows * row_elems;
    if (n == 0 || heur == kMax) return B200_ROI_OK;                     // the running maximum is already the result
    const unsigned blocks = (unsigned)((n + kCombineThreads - 1) / kCombineThreads);
    tta_finish_kernel<<<blocks, kCombineThreads, 0, stream>>>(acc, row_elems, n, row_count, count, heur);
    return finish_launch(1);
}

int b200_resize_width_u8(const unsigned char* src, long long src_pitch, int height, int width, int out_width, unsigned char* dst,
                         b200_stream_t stream) {
    if (!src || !dst || height < 1 || width < 1 || out_width < 1 || src_pitch < 3LL * width) return B200_ROI_EINVAL;
    if ((long long)height * out_width >= (1LL << 31)) return B200_ROI_EINVAL;
    const long long n = (long long)height * out_width;
    const double scale_x = 1.0 / ((double)out_width / width);            // cv2: 1 / inv_scale_x, inv_scale_x = W' / w
    resize_width_u8_kernel<<<(unsigned)((n + kResizeThreads - 1) / kResizeThreads), kResizeThreads, 0, stream>>>(src, src_pitch, height, width,
                                                                                                              out_width, scale_x, dst);
    return finish_launch(1);
}

}  // extern "C"
