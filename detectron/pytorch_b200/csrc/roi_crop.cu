// roi_crop.cu -- RoICrop: bilinear sampling of an NCHW image from an explicit (y,x) grid.
//
// Semantics: lib/model/roi_crop/src/roi_crop_cuda_kernel.cu (reference) getTopLeft :11-22,
// bilinearSamplingFromGrid :47-109, backwardBilinearSampling :111-194: align_corners-style mapping
// (g+1)(size-1)/2, zero padding per tap, RoI b reads image b / (R/N), image gradient by fp32 atomics,
// grid gradient never written (stays zero).  Forward values are bit-identical to the reference.
//
// Layout choice: the sampling geometry of an output pixel is the same for every channel, so one
// thread owns one output pixel (b, y, x), computes its 4 tap offsets + weights once, and walks the
// channel slab; adjacent threads are adjacent x, so output stores are coalesced.
#include "common.cuh"

namespace b200 {

constexpr int kCropThreads = 256;

struct CropTaps {
    int   off;                    // yTop * W + xLeft (may be negative; only used for taps that are in)
    bool  tl, tr, bl, br;
    float w_tl, w_tr, w_bl, w_br;
};

__device__ __forceinline__ void crop_topleft(float g, int size, int& point, float& weight) {
    const float coord = __fmul_rn(__fmul_rn(__fadd_rn(g, 1.f), (float)(size - 1)), 0.5f);
    const float fl = floorf(coord);
    point = (int)fl;
    weight = __fadd_rn(__fsub_rn(fl, coord), 1.f);
}

__device__ __forceinline__ CropTaps crop_taps(const float* __restrict__ g, int H, int W) {
    int yt, xl; float yW, xW;
    crop_topleft(g[1], W, xl, xW);
    crop_topleft(g[0], H, yt, yW);
    const bool xin0 = xl >= 0 && xl <= W - 1, xin1 = xl + 1 >= 0 && xl + 1 <= W - 1;
    const bool yin0 = yt >= 0 && yt <= H - 1, yin1 = yt + 1 >= 0 && yt + 1 <= H - 1;
    CropTaps t;
    t.off = yt * W + xl;
    t.tl = xin0 && yin0; t.tr = xin1 && yin0; t.bl = xin0 && yin1; t.br = xin1 && yin1;
    const float omx = __fsub_rn(1.f, xW), omy = __fsub_rn(1.f, yW);
    t.w_tl = __fmul_rn(xW, yW); t.w_tr = __fmul_rn(omx, yW);
    t.w_bl = __fmul_rn(xW, omy); t.w_br = __fmul_rn(omx, omy);
    return t;
}

template <bool BACKWARD>
__global__ void __launch_bounds__(kCropThreads)
roi_crop_kernel(const float* __restrict__ in,        // fwd: image       bwd: grad_output
                const float* __restrict__ grids,
                float* __restrict__ out,             // fwd: output      bwd: grad_image (pre-zeroed)
                int N, int C, int H, int W, int R, int oh, int ow, int c_per_cta) {
    const int per = R / N;                            // reference :217 roiPerImage = ob / ib
    const long pix = (long)blockIdx.x * kCropThreads + threadIdx.x;   // (b, y, x)
    const long npix = (long)R * oh * ow;
    if (pix >= npix) return;
    const int b = (int)(pix / ((long)oh * ow));
    const int yx = (int)(pix % ((long)oh * ow));
    const CropTaps t = crop_taps(grids + pix * 2, H, W);
    const int c0 = blockIdx.y * c_per_cta, c1 = min(C, c0 + c_per_cta);
    const bool any = t.tl || t.tr || t.bl || t.br;
    const int bi = per > 0 ? b / per : 0;
    const bool img_ok = bi < N;
    for (int c = c0; c < c1; ++c) {
        const size_t oidx = ((size_t)b * C + c) * oh * ow + yx;
        if (!any || !img_ok) {                        // reference `continue`s and leaves the zero-filled output
            if (!BACKWARD) out[oidx] = 0.f;
            continue;
        }
        const long base = ((long)bi * C + c) * H * W + t.off;
        if (!BACKWARD) {
            const float vtl = t.tl ? __ldg(in + base) : 0.f, vtr = t.tr ? __ldg(in + base + 1) : 0.f;
            const float vbl = t.bl ? __ldg(in + base + W) : 0.f, vbr = t.br ? __ldg(in + base + W + 1) : 0.f;
            out[oidx] = __fmaf_rn(t.w_br, vbr, __fmaf_rn(t.w_bl, vbl, __fmaf_rn(t.w_tl, vtl, __fmul_rn(t.w_tr, vtr))));
        } else {
            const float go = in[oidx];
            if (t.tl) atomicAdd(out + base, __fmul_rn(go, t.w_tl));
            if (t.tr) atomicAdd(out + base + 1, __fmul_rn(go, t.w_tr));
            if (t.bl) atomicAdd(out + base + W, __fmul_rn(go, t.w_bl));
            if (t.br) atomicAdd(out + base + W + 1, __fmul_rn(go, t.w_br));
        }
    }
}

static void crop_grid(int C, long npix, dim3& grid, int& cpc) {
    const long xb = (npix + kCropThreads - 1) / kCropThreads;
    cpc = C;
    while (cpc > 4 && xb * ((C + cpc - 1) / cpc) < 8L * kNumSMs) cpc /= 2;
    grid = dim3((unsigned)xb, (unsigned)((C + cpc - 1) / cpc));
}

// ---- backward, vector-reduction path (same idea as roi_align_bwd_nhwc.cu) ------------------------------------------------
// The sampling geometry of an output pixel is the same for every channel, so in a channel-innermost scratch image of the
// gradient every tap updates C contiguous floats: one red.global.add.v4.f32 per tap per FOUR channels (6.4 M vector reductions
// instead of 25.7 M scalar atomics at 512 RoIs x 7 x 7 x 256 channels), 1 KB contiguous per (pixel, tap) across the CTA.
// One CTA per (RoI, <= 256 channels): grad_output[r] (one contiguous block) is staged transposed to [pixel][channel] in shared
// memory; thread = (pixel lane, channel quad).  The scratch image is transposed back to NCHW by the RoIAlign path's kernel.
// Per-tap terms FMUL(go, w) as in the reference (roi_crop_cuda_kernel.cu:163-190); summation order undefined, as with atomicAdd.
constexpr int kCropChunk = 256;

__global__ void __launch_bounds__(256)
roi_crop_bwd_nhwc_scatter(const float* __restrict__ go, const float* __restrict__ grids, float* __restrict__ scratch, int N, int C,
                          int H, int W, int R, int oh, int ow, int c_pad) {
    extern __shared__ __align__(16) float s_go[];             // [pixels][c_pad]
    const int r = blockIdx.x, c0 = blockIdx.y * kCropChunk;
    const int cc = min(kCropChunk, C - c0);
    const int pixels = oh * ow;
    const int per = R / N;
    const int bi = per > 0 ? r / per : 0;
    if (bi >= N) return;
    const float* src = go + ((size_t)r * C + c0) * pixels;
    for (int k = threadIdx.x; k < cc * pixels; k += 256) {      // coalesced read, transposed write ([c][pix] -> [pix][c])
        const int c = k / pixels, p = k - c * pixels;
        s_go[p * c_pad + c] = __ldg(src + k);
    }
    __syncthreads();
    const int quads = cc >> 2;                                  // cc % 4 == 0 on this path
    const int q = threadIdx.x % quads, pl = threadIdx.x / quads, pstep = 256 / quads;
    if (pl >= pstep) return;
    float* img = scratch + (size_t)bi * H * W * C + c0 + 4 * q;
    for (int p = pl; p < pixels; p += pstep) {
        const CropTaps t = crop_taps(grids + ((size_t)r * pixels + p) * 2, H, W);
        const float4 g = *reinterpret_cast<const float4*>(&s_go[p * c_pad + 4 * q]);
#define B200_CROP_TAP(on, delta, WT)                                                                                       \
        if (on) {                                                                                                          \
            float* dst = img + (size_t)(t.off + (delta)) * C;                                                              \
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(__fmul_rn(g.x, WT)), "f"(__fmul_rn(g.y, WT)), \
                         "f"(__fmul_rn(g.z, WT)), "f"(__fmul_rn(g.w, WT)) : "memory");                                      \
        }
        B200_CROP_TAP(t.tl, 0, t.w_tl)
        B200_CROP_TAP(t.tr, 1, t.w_tr)
        B200_CROP_TAP(t.bl, W, t.w_bl)
        B200_CROP_TAP(t.br, W + 1, t.w_br)
#undef B200_CROP_TAP
    }
}

// returns kPathDeclined when the path does not apply
static bool crop_nhwc_applies(int N, int C, int H, int W, int R, int oh, int ow) {
    if ((C & 3) || C < 16 || N <= 0 || R <= 0 || (R % N) != 0) return false;
    const long long taps = 4LL * R * oh * ow * C;
    return taps >= 2LL * N * C * H * W;                        // zero + transpose of the whole image must pay off
}

static int roi_crop_backward_nhwc(const float* grad_output, const float* grids, int N, int C, int H, int W, int R, int oh, int ow,
                                  float* grad_image, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    if (!crop_nhwc_applies(N, C, H, W, R, oh, ow)) return kPathDeclined;
    const int chunk = C < kCropChunk ? C : kCropChunk;
    if (chunk & 3) return kPathDeclined;                                // thread = (pixel lane, quad): 256 / quads pixel lanes, the rest idle
    const int c_pad = chunk + 4;
    const size_t smem = sizeof(float) * (size_t)oh * ow * c_pad;
    if (smem > 200 * 1024) return kPathDeclined;
    const size_t bytes = sizeof(float) * (size_t)N * C * H * W;
    float* scratch = (float*)workspace;
    const bool own = scratch == nullptr || workspace_bytes < bytes;      // no caller scratch: stream-ordered allocation
    if (own && cudaMallocAsync((void**)&scratch, bytes, stream) != cudaSuccess) { (void)cudaGetLastError(); return kPathDeclined; }
    cudaError_t err = cudaMemsetAsync(scratch, 0, bytes, stream);
    if (err == cudaSuccess) err = (cudaError_t)smem_opt_in(roi_crop_bwd_nhwc_scatter, smem);
    if (err == cudaSuccess) {
        dim3 grid(R, (C + kCropChunk - 1) / kCropChunk);
        roi_crop_bwd_nhwc_scatter<<<grid, 256, smem, stream>>>(grad_output, grids, scratch, N, C, H, W, R, oh, ow, c_pad);
        launch_nhwc_to_nchw(scratch, grad_image, N, C, H * W, stream);
    }
    if (own) cudaFreeAsync(scratch, stream);
    if (err != cudaSuccess) return (int)err;
    return finish_launch(2);
}

}  // namespace b200

using namespace b200;

extern "C" {

int b200_roi_crop_forward(const float* image, const float* grids, int N, int C, int H, int W, int R, int oh, int ow,
                          float* output, b200_stream_t stream) {
    if (N < 0 || C < 0 || H <= 0 || W <= 0 || R < 0 || oh < 0 || ow < 0) return B200_ROI_EINVAL;
    if ((size_t)R * oh * ow * C > 0 && (!image || !grids || !output)) return B200_ROI_EINVAL;
    const long npix = (long)R * oh * ow;
    if (npix == 0 || C == 0) return B200_ROI_OK;
    if (N <= 0) return B200_ROI_EINVAL;
    dim3 grid; int cpc;
    crop_grid(C, npix, grid, cpc);
    roi_crop_kernel<false><<<grid, kCropThreads, 0, stream>>>(image, grids, output, N, C, H, W, R, oh, ow, cpc);
    return finish_launch();
}

size_t b200_roi_crop_backward_workspace_bytes(int N, int C, int H, int W, int R, int oh, int ow) {
    if (N <= 0 || C <= 0 || H <= 0 || W <= 0 || R <= 0 || oh <= 0 || ow <= 0) return 0;
    if (option_get(kOptBwdPath) == 'g' || !crop_nhwc_applies(N, C, H, W, R, oh, ow)) return 0;
    return (sizeof(float) * (size_t)N * C * H * W + 255) / 256 * 256;
}

int b200_roi_crop_backward_ws(const float* grad_output, const float* grids, int N, int C, int H, int W, int R, int oh, int ow,
                              float* grad_image, float* grad_grids, void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    if (N < 0 || C < 0 || H <= 0 || W <= 0 || R < 0 || oh < 0 || ow < 0) return B200_ROI_EINVAL;
    if ((size_t)N * C == 0) return B200_ROI_OK;
    if (!grad_image) return B200_ROI_EINVAL;
    if ((size_t)R * oh * ow > 0 && (!grad_output || !grids)) return B200_ROI_EINVAL;
    if (grad_grids != nullptr) {
        const cudaError_t e0 = cudaMemsetAsync(grad_grids, 0, sizeof(float) * (size_t)R * oh * ow * 2, stream);
        if (e0 != cudaSuccess) return (int)e0;
    }
    if ((long)R * oh * ow > 0 && C > 0 && option_get(kOptBwdPath) != 'g') {      // B200_ROI_ALIGN_BWD_PATH=generic: scalar atomics (A/B)
        const int rc = roi_crop_backward_nhwc(grad_output, grids, N, C, H, W, R, oh, ow, grad_image, workspace, workspace_bytes, stream);
        if (rc != kPathDeclined) return rc;
    }
    cudaError_t err = cudaMemsetAsync(grad_image, 0, sizeof(float) * (size_t)N * C * H * W, stream);
    if (err != cudaSuccess) return (int)err;
    int launches = 1;
    grad_grids = nullptr;                                       // already zeroed above
    if (grad_grids != nullptr) {
        err = cudaMemsetAsync(grad_grids, 0, sizeof(float) * (size_t)R * oh * ow * 2, stream);
        if (err != cudaSuccess) return (int)err;
        ++launches;
    }
    const long npix = (long)R * oh * ow;
    if (npix == 0 || C == 0) return B200_ROI_OK;
    if (N <= 0) return B200_ROI_EINVAL;
    dim3 grid; int cpc;
    crop_grid(C, npix, grid, cpc);
    roi_crop_kernel<true><<<grid, kCropThreads, 0, stream>>>(grad_output, grids, grad_image, N, C, H, W, R, oh, ow, cpc);
    (void)launches;
    return finish_launch();
}


int b200_roi_crop_backward(const float* grad_output, const float* grids, int N, int C, int H, int W, int R, int oh, int ow,
                           float* grad_image, float* grad_grids, b200_stream_t stream) {
    return b200_roi_crop_backward_ws(grad_output, grids, N, C, H, W, R, oh, ow, grad_image, grad_grids, nullptr, 0, stream);
}

}  // extern "C"
