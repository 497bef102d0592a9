// roi_align_bwd_nhwc.cu -- Caffe2-exact RoIAlign BACKWARD, vector-reduction path.
//
// The reference backward (and our generic one) issues one fp32 atomic per tap per channel:
// 102.8 M scalar reductions at BASELINE cfg2, bound by the L2 atomic unit.  A 16-byte
// `red.global.add.v4.f32` costs the same L2 slot as a scalar one (tools/ubench_red.cu measures it), i.e. 4x the floats per op when
// the four addends are adjacent in memory.  In NCHW nothing adjacent is ever updated together, but
// the sampling geometry is identical for every channel, so in a channel-innermost (NHWC) image of
// dX each tap updates C contiguous floats.  Hence:
//
//   1. zero an NHWC scratch image of dX (workspace, same size as dX);
//   2. one CTA per (RoI, <=256 channels): stage dY[r] (one contiguous block) into shared memory
//      transposed to [bin][channel]; lane = (sample of a 4-sample group, 4-channel group); every tap is
//      one red.global.add.v4.f32 -- 25.7 M vector reductions instead of 102.8 M scalar ones;
//   3. transpose the scratch image back to NCHW through shared memory (both sides coalesced).
//
// The per-tap terms are the reference's, rounded identically: g_k = FMUL(top, w_k) / count
// (roi_align_kernel.cu:252-255; count is a power of two on this path so the division is an exact
// scaling).  Summation order is undefined, exactly as with the reference's atomicAdd.
//
// Semantics: lib/modeling/roi_xfrom/roi_align/src/roi_align_kernel.cu (reference) :150-193, :195-270.
#include "common.cuh"

namespace b200 {

constexpr int kBwThreads = 256;
constexpr int kBwChunk = 256;             // channels per CTA
constexpr int kBwAxisMax = 32;            // P * sr per axis

struct __align__(16) BwAxis {
    int   low;      // low cell
    int   valid;
    float l, h;
};

__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

template <int SR>
__global__ void __launch_bounds__(kBwThreads)
roi_align_bwd_nhwc_scatter(const float* __restrict__ top_diff, const float* __restrict__ rois, float* __restrict__ scratch,
                           float scale, int N, int C, int H, int W, int PH, int PW, int c_pad, const int* __restrict__ row_map) {
    extern __shared__ __align__(16) float s_dy[];          // [bins][c_pad]   (c_pad = chunk + 4, multiple of 4)
    __shared__ BwAxis s_y[kBwAxisMax], s_x[kBwAxisMax];
    const int r = blockIdx.x;
    const int c0 = blockIdx.y * kBwChunk;
    const int cc = min(kBwChunk, C - c0);                  // channels of this CTA
    const int bins = PH * PW;
    const int ny = PH * SR, nx = PW * SR;
    const int tid = threadIdx.x;

    const XfromRoi g = xfrom_roi(rois + 5 * (size_t)r, scale, PH, PW, SR);
    if (g.batch < 0 || g.batch >= N) return;               // reference would scatter out of bounds; defined here as no-op
    if (tid < ny + nx) {
        const bool isy = tid < ny;
        const int s = isy ? tid : tid - ny;
        const AxisTap a = isy ? xfrom_axis(xfrom_coord(g.start_h, g.bin_h, s / SR, s % SR, SR), H)
                              : xfrom_axis(xfrom_coord(g.start_w, g.bin_w, s / SR, s % SR, SR), W);
        BwAxis e; e.low = a.low; e.valid = a.valid ? 1 : 0; e.l = a.l; e.h = a.h;
        if (isy) s_y[s] = e; else s_x[s] = e;
    }
    // stage dY[r, c0:c0+cc, :, :] (contiguous cc*bins floats) transposed to [bin][channel]
    const float* src = top_diff + ((size_t)(row_map ? row_map[r] : r) * C + c0) * bins;
    for (int idx = tid; idx < cc * bins; idx += kBwThreads) {
        const int c = idx / bins, b = idx - c * bins;
        s_dy[b * c_pad + c] = __ldg(src + idx);
    }
    __syncthreads();

    // lane = (q: sample of a 4-sample group, i: 4-channel group of a 32-channel slab)
    const int lane = tid & 31, warp = tid >> 5, q = lane >> 3, i = lane & 7;
    const int nsamp = ny * nx;
    const int slabs = (cc + 31) / 32;
    float* img = scratch + (size_t)g.batch * H * W * C + c0;
    constexpr float kInv = 1.f / (float)(SR * SR);
    for (int item = warp; item < ((nsamp + 3) / 4) * slabs; item += kBwThreads / 32) {
        const int sg = item / slabs, slab = item - sg * slabs;
        const int s = sg * 4 + q;
        const int c = slab * 32 + 4 * i;
        if (s >= nsamp || c >= cc) continue;
        const int sy = s / nx, sx = s - sy * nx;
        const BwAxis ey = s_y[sy], ex = s_x[sx];
        if (!ey.valid || !ex.valid) continue;
        const int bin = (sy / SR) * PW + (sx / SR);
        const float4 t = *reinterpret_cast<const float4*>(s_dy + bin * c_pad + c);
        const float w1 = __fmul_rn(ey.h, ex.h), w2 = __fmul_rn(ey.h, ex.l);
        const float w3 = __fmul_rn(ey.l, ex.h), w4 = __fmul_rn(ey.l, ex.l);
        // the high taps coincide with the low ones at the map border (reference: x_high = x_low = W-1)
        const int yh = min(ey.low + 1, H - 1), xh = min(ex.low + 1, W - 1);
        float* p11 = img + ((size_t)ey.low * W + ex.low) * C + c;
        float* p12 = img + ((size_t)ey.low * W + xh) * C + c;
        float* p21 = img + ((size_t)yh * W + ex.low) * C + c;
        float* p22 = img + ((size_t)yh * W + xh) * C + c;
        const bool vec = (cc - c >= 4) && ((C & 3) == 0);
#define B200_TERM(v, w) (SR == 3 ? __fdiv_rn(__fmul_rn(v, w), 9.f) : __fmul_rn(__fmul_rn(v, w), kInv))
        if (vec) {
            red_add_v4(p11, B200_TERM(t.x, w1), B200_TERM(t.y, w1), B200_TERM(t.z, w1), B200_TERM(t.w, w1));
            red_add_v4(p12, B200_TERM(t.x, w2), B200_TERM(t.y, w2), B200_TERM(t.z, w2), B200_TERM(t.w, w2));
            red_add_v4(p21, B200_TERM(t.x, w3), B200_TERM(t.y, w3), B200_TERM(t.z, w3), B200_TERM(t.w, w3));
            red_add_v4(p22, B200_TERM(t.x, w4), B200_TERM(t.y, w4), B200_TERM(t.z, w4), B200_TERM(t.w, w4));
        } else {
            const float tv[4] = {t.x, t.y, t.z, t.w};
            for (int k = 0; k < 4 && c + k < cc; ++k) {
                atomicAdd(p11 + k, B200_TERM(tv[k], w1)); atomicAdd(p12 + k, B200_TERM(tv[k], w2));
                atomicAdd(p21 + k, B200_TERM(tv[k], w3)); atomicAdd(p22 + k, B200_TERM(tv[k], w4));
            }
        }
#undef B200_TERM
    }
}

// scratch (N, H*W, C)  ->  dX (N, C, H*W): 32 x 32 tiles through shared memory, both sides coalesced
__global__ void __launch_bounds__(256)
nhwc_to_nchw_kernel(const float* __restrict__ scratch, float* __restrict__ dx, int C, int HW) {
    __shared__ float t[32][33];
    const int n = blockIdx.z;
    const int p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, tyy = threadIdx.x >> 5;          // 32 x 8
    const float* src = scratch + (size_t)n * HW * C;
    float* dst = dx + (size_t)n * C * HW;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int p = p0 + tyy + 8 * k, c = c0 + tx;
        t[tyy + 8 * k][tx] = (p < HW && c < C) ? __ldg(src + (size_t)p * C + c) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int c = c0 + tyy + 8 * k, p = p0 + tx;
        if (c < C && p < HW) dst[(size_t)c * HW + p] = t[tx][tyy + 8 * k];
    }
}

// shared with the RoICrop backward (roi_crop.cu)
void launch_nhwc_to_nchw(const float* scratch, float* dx, int N, int C, int HW, cudaStream_t stream) {
    dim3 tgrid((HW + 31) / 32, (C + 31) / 32, N);
    nhwc_to_nchw_kernel<<<tgrid, 256, 0, stream>>>(scratch, dx, C, HW);
}

size_t roi_align_bwd_nhwc_workspace_bytes(int N, int C, int H, int W) {
    return ((size_t)N * C * H * W * sizeof(float) + 255) / 256 * 256;
}

// returns kPathDeclined when the path does not apply (caller falls back to the generic scalar-atomic kernel)
int roi_align_backward_nhwc(const float* top_diff, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                            const float* rois, float* bottom_diff, const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    if (sr < 1 || sr > 4 || PH * sr > kBwAxisMax || PW * sr > kBwAxisMax) return kPathDeclined;
    if (workspace == nullptr || workspace_bytes < roi_align_bwd_nhwc_workspace_bytes(N, C, H, W)) return kPathDeclined;
    if (R <= 0 || C <= 0 || N <= 0) return kPathDeclined;
    float* scratch = (float*)workspace;
    cudaError_t err = cudaMemsetAsync(scratch, 0, sizeof(float) * (size_t)N * C * H * W, stream);
    if (err != cudaSuccess) return (int)err;
    const int chunk = C < kBwChunk ? C : kBwChunk;
    const int c_pad = ((chunk + 3) / 4) * 4 + 4;
    const size_t smem = sizeof(float) * (size_t)PH * PW * c_pad;
    if (smem > 200 * 1024) return kPathDeclined;
    dim3 grid(R, (C + kBwChunk - 1) / kBwChunk);
    const auto scatter = sr == 1 ? roi_align_bwd_nhwc_scatter<1> : sr == 2 ? roi_align_bwd_nhwc_scatter<2>
                       : sr == 3 ? roi_align_bwd_nhwc_scatter<3> : roi_align_bwd_nhwc_scatter<4>;
    if (const int rc = smem_opt_in(scatter, smem)) return rc;
    scatter<<<grid, kBwThreads, smem, stream>>>(top_diff, rois, scratch, scale, N, C, H, W, PH, PW, c_pad, row_map);
    const int HW = H * W;
    dim3 tgrid((HW + 31) / 32, (C + 31) / 32, N);
    nhwc_to_nchw_kernel<<<tgrid, 256, 0, stream>>>(scratch, bottom_diff, C, HW);
    return finish_launch(2);
}

}  // namespace b200
