// roi_align_legacy.cu -- the legacy (jwyang-style) RoIAlign: ONE bilinear sample at each of the
// aligned_h x aligned_w lattice corners of the RoI, with part of the interpolation carried in fp64
// because of the `1.` literals in the reference source.
//
// Semantics: lib/model/roi_align/src/roi_align_kernel.cu (reference) ROIAlignForward :15-70,
// ROIAlignBackward :94-143.  The mixed fp32/fp64 rounding recipe below is the one nvcc emits for
// the reference (see oracle/roi_ops_oracle.c, "RoIAlign, legacy variant").
//
// One departure from the reference: maps with a single row or column.  The reference takes the first tap at
// hstart = min(floor(h), H - 2) and the second at hstart + 1, so on H = 1 every in-map sample reads (forward) and
// atomically adds to (backward) row -1 -- before the tensor, or in the previous channel plane -- and likewise column -1
// on W = 1.  Small images give such maps at the top pyramid levels, so here the first tap is clamped to
// max(min(floor(h), H - 2), 0) and the second to min(hstart + 1, H - 1) (same for w): on a one-row map both taps are
// row 0, the convention of the Caffe2-style RoIAlign on its clamped last row.  The weights are left as computed, so
// the forward gives the row's value and the backward puts the whole gradient on row 0.  For H, W >= 2 the clamps
// change nothing and the results stay bit-identical to the reference.
//
// Layout choice: one CTA per (RoI, channel slab); the P x P lattice geometry (cell index + the two
// ratios) is computed once per CTA into shared memory instead of once per output element.
#include "common.cuh"

namespace b200 {

constexpr int kLegThreads = 256;
constexpr int kLegTabMax = 1024;   // lattice points cached per CTA (P*P); larger lattices compute on the fly

struct __align__(16) LegPoint {
    int   off;       // hstart * W + wstart, or -1 if the point is outside the map
    float hr, wr;    // h_ratio, w_ratio
    int   taps;      // bit 0: the right taps are column wstart + 1 (else wstart); bit 1: the lower taps are row hstart + 1
};

__device__ __forceinline__ LegPoint legacy_point(const float* __restrict__ roi, float scale, int PH, int PW,
                                                 int H, int W, int ph, int pw) {
    const float sw = __fmul_rn(roi[1], scale), sh = __fmul_rn(roi[2], scale);
    const float rw = fmaxf(__fadd_rn(__fmaf_rn(roi[3], scale, -sw), 1.f), 0.f);
    const float rh = fmaxf(__fadd_rn(__fmaf_rn(roi[4], scale, -sh), 1.f), 0.f);
    const float bh = (float)__ddiv_rn((double)rh, __dsub_rn((double)PH, 1.));
    const float bw = (float)__ddiv_rn((double)rw, __dsub_rn((double)PW, 1.));
    const float h = __fmaf_rn((float)ph, bh, sh);
    const float w = __fmaf_rn((float)pw, bw, sw);
    LegPoint p;
    if (h < 0 || h >= (float)H || w < 0 || w >= (float)W) {
        p.off = -1; p.hr = 0.f; p.wr = 0.f; p.taps = 0;
        return p;
    }
    const int hs = (int)fmaxf(fminf(floorf(h), (float)(H - 2)), 0.f);   // 0 on a one-row map (the reference: -1)
    const int ws = (int)fmaxf(fminf(floorf(w), (float)(W - 2)), 0.f);
    p.off = hs * W + ws;
    p.taps = (ws + 1 <= W - 1 ? 1 : 0) | (hs + 1 <= H - 1 ? 2 : 0);
    p.hr = __fsub_rn(h, (float)hs);
    p.wr = __fsub_rn(w, (float)ws);
    return p;
}

template <bool BACKWARD>
__global__ void __launch_bounds__(kLegThreads)
roi_align_legacy_kernel(const float* __restrict__ in, const float* __restrict__ rois, float* __restrict__ out,
                        float scale, int N, int C, int H, int W, int PH, int PW, int c_per_cta) {
    __shared__ LegPoint tab[kLegTabMax];
    const int n = blockIdx.x;
    const int c0 = blockIdx.y * c_per_cta, c1 = min(C, c0 + c_per_cta);
    const float* roi = rois + 5 * (size_t)n;
    const int bins = PH * PW;
    const bool use_tab = bins <= kLegTabMax;
    if (use_tab)
        for (int b = threadIdx.x; b < bins; b += kLegThreads) tab[b] = legacy_point(roi, scale, PH, PW, H, W, b / PW, b % PW);
    __syncthreads();

    // the reference keeps the batch index as float: img_start = (int)(b * C * H * W)  (:51, :126)
    const float bf = roi[0];
    const long long img_start = (long long)(int)__fmul_rn(__fmul_rn(__fmul_rn(bf, (float)C), (float)H), (float)W);
    const bool batch_ok = (bf >= 0.f) && ((int)bf < N);
    const int total = (c1 - c0) * bins;
    for (int idx = threadIdx.x; idx < total; idx += kLegThreads) {
        const int c = c0 + idx / bins, bin = idx % bins;
        const size_t oidx = ((size_t)n * C + c) * bins + bin;
        const LegPoint p = use_tab ? tab[bin] : legacy_point(roi, scale, PH, PW, H, W, bin / PW, bin % PW);
        if (p.off < 0 || !batch_ok) {
            if (!BACKWARD) out[oidx] = 0.f;
            continue;
        }
        const size_t ul = (size_t)(img_start + (long long)c * H * W + p.off);
        const size_t ur = ul + (p.taps & 1), dl = ul + (p.taps & 2 ? W : 0), dr = dl + (p.taps & 1);
        if (!BACKWARD) {
            const float vul = __ldg(in + ul), vur = __ldg(in + ur), vdl = __ldg(in + dl), vdr = __ldg(in + dr);
            const double omh = __dsub_rn(1.0, (double)p.hr), omw = __dsub_rn(1.0, (double)p.wr);
            const double t_ur = __dmul_rn((double)p.wr, __dmul_rn(omh, (double)vur));
            double acc = __fma_rn(__dmul_rn((double)vul, omh), omw, t_ur);
            acc = __fma_rn(omw, (double)__fmul_rn(p.hr, vdl), acc);
            acc = __dadd_rn(acc, (double)__fmul_rn(p.wr, __fmul_rn(p.hr, vdr)));
            out[oidx] = (float)acc;
        } else {
            const float g = in[oidx];
            const double gomh = __dmul_rn((double)g, __dsub_rn(1.0, (double)p.hr));
            const float omw = __fsub_rn(1.f, p.wr);
            const float ghr = __fmul_rn(p.hr, g);
            atomicAdd(out + ul, (float)__dmul_rn(gomh, (double)omw));
            atomicAdd(out + ur, (float)__dmul_rn(gomh, (double)p.wr));
            atomicAdd(out + dl, __fmul_rn(omw, ghr));
            atomicAdd(out + dr, __fmul_rn(p.wr, ghr));
        }
    }
}

static int legacy_c_per_cta(int R, int C, int bins) {
    int cpc = C;
    while (cpc > 1 && (long)R * ((C + cpc - 1) / cpc) < 8L * kNumSMs && (cpc / 2) * bins >= kLegThreads) cpc /= 2;
    return cpc;
}

int roi_align_legacy_forward(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW,
                             const float* rois, float* top, cudaStream_t stream) {
    if (R == 0 || C == 0) return B200_ROI_OK;
    const int cpc = legacy_c_per_cta(R, C, PH * PW);
    dim3 grid(R, (C + cpc - 1) / cpc);
    roi_align_legacy_kernel<false><<<grid, kLegThreads, 0, stream>>>(bottom, rois, top, scale, N, C, H, W, PH, PW, cpc);
    return finish_launch();
}

int roi_align_legacy_backward(const float* top_diff, float scale, int N, int R, int H, int W, int C, int PH, int PW,
                              const float* rois, float* bottom_diff, cudaStream_t stream) {
    cudaError_t err = cudaMemsetAsync(bottom_diff, 0, sizeof(float) * (size_t)N * C * H * W, stream);
    if (err != cudaSuccess) return (int)err;
    if (R == 0 || C == 0) return B200_ROI_OK;
    const int cpc = legacy_c_per_cta(R, C, PH * PW);
    dim3 grid(R, (C + cpc - 1) / cpc);
    roi_align_legacy_kernel<true><<<grid, kLegThreads, 0, stream>>>(top_diff, rois, bottom_diff, scale, N, C, H, W, PH, PW, cpc);
    return finish_launch();
}

}  // namespace b200
