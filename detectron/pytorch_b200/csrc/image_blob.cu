// image_blob.cu -- the network's input `data` blob (lib/utils/blob.py:37-148 get_image_blob / prep_im_for_blob /
// im_list_to_blob, lib/roi_data/minibatch.py:47-79 _get_image_blob, lib/roi_data/loader.py:251-260 pad_image_data) for all
// images of a call in one launch, from the decoded uint8 BGR images.
//
// Per image: flip (im[:, ::-1, :]) -> float32 - PIXEL_MEANS (numpy: float32(float64(v) - mean), a (3, 256) table) ->
// cv2.resize(fx = fy = s, INTER_LINEAR) with IPP off -> zero padding to the blob size -> NCHW.
//   Linear: per axis cv2_linear_tap (common.cuh) with cv2's scale 1 / s; the horizontal pass S[s0] * a0 + S[s1] * a1 on both
//   source rows, then D0 * b0 + D1 * b1; every product and sum rounded on its own (_rn intrinsics).  A flipped image uses the
//   taps of the flipped frame and reads the physical column W - 1 - s.
//   Exact 2x shrink (1 / s == 2.0): cv2's fast INTER_AREA, for 3 channels its scalar loop (((a00 + a01) + a10) + a11) * .25.
//   On an odd side the last row / column averages the taps inside the image: (a + b) * .5, or a00 at the corner.
//
// Work layout: one thread per (image, blob row, 4 consecutive blob columns); it writes all 3 channel planes, one 16-byte store
// each (scalar stores when blob_w % 4 != 0, which happens only without FPN padding).  Every element of the blob is written
// once, padding included.  Source bytes go through the read-only path; an image is 1-6 MB and stays in L2.  The bound is the
// blob's HBM write traffic, N * 3 * Hp * Wp * 4 bytes.
#include "common.cuh"

namespace b200 {

namespace {
constexpr int kBlobThreads = 256;

struct Px {
    float c[3];
};

// pixel (y, x) of the (possibly flipped) image, minus the means
__device__ __forceinline__ Px load_px(const unsigned char* __restrict__ row, int x, const b200_image_blob_desc& d, const float* tab) {
    const int px = d.flipped ? d.width - 1 - x : x;
    const unsigned char* p = row + 3LL * px;
    Px v;
#pragma unroll
    for (int c = 0; c < 3; ++c) v.c[c] = tab[c * 256 + __ldg(p + c)];
    return v;
}

__device__ __forceinline__ Px linear_value(const unsigned char* __restrict__ r0, const unsigned char* __restrict__ r1, const Cv2Tap& tx,
                                           const Cv2Tap& ty, const b200_image_blob_desc& d, const float* tab) {
    const Px p00 = load_px(r0, tx.s0, d, tab), p01 = load_px(r0, tx.s1, d, tab);
    const Px p10 = load_px(r1, tx.s0, d, tab), p11 = load_px(r1, tx.s1, d, tab);
    Px o;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float d0 = __fadd_rn(__fmul_rn(p00.c[c], tx.w0), __fmul_rn(p01.c[c], tx.w1));
        const float d1 = __fadd_rn(__fmul_rn(p10.c[c], tx.w0), __fmul_rn(p11.c[c], tx.w1));
        o.c[c] = __fadd_rn(__fmul_rn(d0, ty.w0), __fmul_rn(d1, ty.w1));
    }
    return o;
}

// cv2's resizeAreaFast at 2x for output pixel (oy, ox): rows 2 oy, 2 oy + 1, columns 2 ox, 2 ox + 1, those past the end dropped
__device__ __forceinline__ Px area_value(const unsigned char* __restrict__ src, int oy, int ox, const b200_image_blob_desc& d,
                                         const float* tab) {
    const int y0 = 2 * oy, x0 = 2 * ox;
    const bool has_y1 = y0 + 1 < d.height, has_x1 = x0 + 1 < d.width;
    const unsigned char* r0 = src + (long long)y0 * d.row_pitch;
    const unsigned char* r1 = has_y1 ? r0 + d.row_pitch : r0;
    const int x1 = has_x1 ? x0 + 1 : x0;
    const Px a00 = load_px(r0, x0, d, tab), a01 = load_px(r0, x1, d, tab);
    const Px a10 = load_px(r1, x0, d, tab), a11 = load_px(r1, x1, d, tab);
    Px o;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        if (has_y1 && has_x1)
            o.c[c] = __fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(a00.c[c], a01.c[c]), a10.c[c]), a11.c[c]), .25f);
        else if (has_y1)
            o.c[c] = __fmul_rn(__fadd_rn(a00.c[c], a10.c[c]), .5f);
        else if (has_x1)
            o.c[c] = __fmul_rn(__fadd_rn(a00.c[c], a01.c[c]), .5f);
        else
            o.c[c] = a00.c[c];
    }
    return o;
}

// grid: x over (blob row, 4-column group) of one image, y = descriptor index
__global__ void __launch_bounds__(kBlobThreads)
image_blob_kernel(const unsigned char* __restrict__ src_base, const b200_image_blob_desc* __restrict__ descs,
                  const float* __restrict__ mean_table, int Hp, int Wp, bool vec, float* __restrict__ out) {
    __shared__ float tab[3 * 256];
    for (int i = threadIdx.x; i < 3 * 256; i += kBlobThreads) tab[i] = __ldg(mean_table + i);
    __syncthreads();
    const b200_image_blob_desc d = descs[blockIdx.y];
    const int Wq = (Wp + 3) >> 2;
    const long long t = (long long)blockIdx.x * kBlobThreads + threadIdx.x;
    if (t >= (long long)Hp * Wq) return;
    const int y = (int)(t / Wq), x0 = (int)(t % Wq) * 4;
    const int oh = min(d.out_h, Hp), ow = min(d.out_w, Wp);
    const unsigned char* src = src_base + d.src_offset;
    const bool row_in = y < oh && d.height > 0 && d.width > 0;
    Cv2Tap ty{};
    const unsigned char *r0 = src, *r1 = src;
    if (row_in && !d.area2x) {
        ty = cv2_linear_tap(y, d.inv_scale, d.height, false);
        r0 = src + (long long)ty.s0 * d.row_pitch;
        r1 = src + (long long)ty.s1 * d.row_pitch;
    }
    float v[3][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int x = x0 + j;
        Px p{{0.f, 0.f, 0.f}};
        if (row_in && x < ow)
            p = d.area2x ? area_value(src, y, x, d, tab) : linear_value(r0, r1, cv2_linear_tap(x, d.inv_scale, d.width, true), ty, d, tab);
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c][j] = p.c[c];
    }
    const long long plane = (long long)Hp * Wp;
    float* o = out + (long long)d.slot * 3 * plane + (long long)y * Wp + x0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float* oc = o + c * plane;
        if (vec) {
            *reinterpret_cast<float4*>(oc) = make_float4(v[c][0], v[c][1], v[c][2], v[c][3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (x0 + j < Wp) oc[j] = v[c][j];
        }
    }
}
}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_image_blob(const unsigned char* src, const b200_image_blob_desc* descs, int num_images, const float* mean_table, int blob_h,
                    int blob_w, float* out, b200_stream_t stream) {
    if (!src || !descs || !mean_table || !out) return B200_ROI_EINVAL;
    if (num_images < 1 || num_images > 65535 || blob_h < 1 || blob_w < 1 || (long long)blob_h * blob_w >= (1LL << 31)) return B200_ROI_EINVAL;
    const bool vec = blob_w % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0;
    const long long groups = (long long)blob_h * ((blob_w + 3) / 4);
    const dim3 grid((unsigned)((groups + kBlobThreads - 1) / kBlobThreads), (unsigned)num_images);
    image_blob_kernel<<<grid, kBlobThreads, 0, stream>>>(src, descs, mean_table, blob_h, blob_w, vec, out);
    return finish_launch(1);
}

}  // extern "C"
