/*
 * oracle/roi_ops_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement (plain C, fp32 op-for-op) of the reference's CUDA kernels for the
 * RoIAlign / RoIPool / RoICrop / NMS hot path.  The reference (roytseng-tw/Detectron.pytorch)
 * ships NO CPU RoIAlign and NO tests/golden vectors, so every function here follows the
 * reference *.cu kernel it cites, including the exact FMA contraction that
 * `nvcc 12.9 -gencode arch=compute_100a,code=sm_100a` (default -fmad=true) emits for it
 * (read from `cuobjdump -sass`; recipes are noted at each function).  Build with
 * `-ffp-contract=off` so that ONLY the explicitly written fmaf()/fma() calls fuse.
 *
 * Pinning status: the reference holds no golden vectors (SURVEY.md 8c).  This oracle is pinned
 * against (a) outputs of the reference's own kernels recompiled unmodified for sm_100a
 * (oracle/_ref; fixtures + generating script under tests/golden/) and
 * (b) torchvision.ops.roi_align(aligned=False)/roi_pool and F.grid_sample on CPU
 * (tests/test_oracle.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this file's shared object.  The product path never does.
 *
 * All tensors are dense row-major ("contiguous") fp32 unless noted.
 */
#include <math.h>
#include <float.h>
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define ORACLE_API __attribute__((visibility("default")))

ORACLE_API void oracle_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

ORACLE_API int oracle_max_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* ------------------------------------------------------------------------------------------
 * RoIAlign, Caffe2-exact variant ("xfrom")
 * reference: lib/modeling/roi_xfrom/roi_align/src/roi_align_kernel.cu
 *   bilinear_interpolate          :16-63
 *   ROIAlignForward               :65-121
 *   bilinear_interpolate_gradient :150-193
 *   ROIAlignBackward              :195-270
 * SASS recipe (sm_100a):
 *   start      = FMUL(x1, scale)
 *   roi_width  = FMNMX(FFMA(x2, scale, -start), 1)        (end is never rounded on its own)
 *   bin        = roi_width / P                            (IEEE RN division)
 *   grid       = sr > 0 ? sr : (int)ceilf(bin)
 *   base(p)    = FFMA((float)p, bin, start)
 *   coord      = FADD(base, FMUL((float)i + .5f, bin) / (float)grid)
 *   val        = FFMA(v4,w4, FFMA(v3,w3, FFMA(v1,w1, FMUL(v2,w2))))
 *   out        = (sum over iy, ix in order) / (float)(grid_h*grid_w)
 * ------------------------------------------------------------------------------------------ */

/* g_fused = 1 (default): the FMA contraction nvcc emits for the reference kernel (what the GPU
 * reference computes).  g_fused = 0: every product/sum rounded separately (strict C semantics of
 * the source text) -- this variant is bit-identical to torchvision.ops.roi_align(aligned=False)
 * on CPU and is used only to pin the index/weight logic against that independent implementation. */
static int g_fused = 1;
ORACLE_API void oracle_set_fused(int fused) { g_fused = fused; }

typedef struct {
    int   y_low, y_high, x_low, x_high;   /* -1 when the sample is outside the map */
    float w1, w2, w3, w4;
} tap_t;

static inline void xfrom_roi_geometry(const float* roi, float scale, int PH, int PW, int sr,
                                      int* batch, float* start_w, float* start_h,
                                      float* bin_w, float* bin_h, int* grid_w, int* grid_h) {
    *batch = (int)roi[0];
    float sw = roi[1] * scale;
    float sh = roi[2] * scale;
    float rw = fmaxf(g_fused ? fmaf(roi[3], scale, -sw) : (roi[3] * scale - sw), 1.f);
    float rh = fmaxf(g_fused ? fmaf(roi[4], scale, -sh) : (roi[4] * scale - sh), 1.f);
    *start_w = sw;
    *start_h = sh;
    *bin_h = rh / (float)PH;
    *bin_w = rw / (float)PW;
    *grid_h = (sr > 0) ? sr : (int)ceilf(*bin_h);
    *grid_w = (sr > 0) ? sr : (int)ceilf(*bin_w);
}

static inline float xfrom_coord(float start, float bin, int p, int i, int grid) {
    float base = g_fused ? fmaf((float)p, bin, start) : (start + (float)p * bin);
    float off = (((float)i + .5f) * bin) / (float)grid;
    return base + off;
}

/* reference :150-193 (and :16-48 for the forward, same index logic) */
static inline void xfrom_taps(int H, int W, float y, float x, tap_t* t) {
    if (y < -1.0f || y > (float)H || x < -1.0f || x > (float)W) {
        t->w1 = t->w2 = t->w3 = t->w4 = 0.f;
        t->x_low = t->x_high = t->y_low = t->y_high = -1;
        return;
    }
    if (y <= 0) y = 0;
    if (x <= 0) x = 0;
    int y_low = (int)y, x_low = (int)x, y_high, x_high;
    if (y_low >= H - 1) { y_high = y_low = H - 1; y = (float)y_low; } else { y_high = y_low + 1; }
    if (x_low >= W - 1) { x_high = x_low = W - 1; x = (float)x_low; } else { x_high = x_low + 1; }
    float ly = y - (float)y_low, lx = x - (float)x_low;
    float hy = 1.f - ly, hx = 1.f - lx;
    t->y_low = y_low; t->y_high = y_high; t->x_low = x_low; t->x_high = x_high;
    t->w1 = hy * hx; t->w2 = hy * lx; t->w3 = ly * hx; t->w4 = ly * lx;
}

ORACLE_API void oracle_roi_align_forward(const float* bottom, const float* rois, int N, int C, int H, int W,
                                         int R, int PH, int PW, float scale, int sr, float* top) {
    (void)N;
#pragma omp parallel for schedule(dynamic, 1)
    for (int n = 0; n < R; ++n) {
        int b, gh, gw; float sw, sh, bw, bh;
        xfrom_roi_geometry(rois + 5 * n, scale, PH, PW, sr, &b, &sw, &sh, &bw, &bh, &gw, &gh);
        const float count = (float)(gh * gw);
        /* taps are channel independent: compute once per (ph,pw,iy,ix) */
        tap_t* taps = (tap_t*)malloc(sizeof(tap_t) * (size_t)PH * PW * gh * gw);
        for (int ph = 0; ph < PH; ++ph)
            for (int pw = 0; pw < PW; ++pw)
                for (int iy = 0; iy < gh; ++iy) {
                    float y = xfrom_coord(sh, bh, ph, iy, gh);
                    for (int ix = 0; ix < gw; ++ix) {
                        float x = xfrom_coord(sw, bw, pw, ix, gw);
                        xfrom_taps(H, W, y, x, &taps[(((size_t)ph * PW + pw) * gh + iy) * gw + ix]);
                    }
                }
        for (int c = 0; c < C; ++c) {
            const float* plane = bottom + ((size_t)b * C + c) * H * W;
            float* out = top + ((size_t)n * C + c) * PH * PW;
            for (int ph = 0; ph < PH; ++ph)
                for (int pw = 0; pw < PW; ++pw) {
                    const tap_t* t = &taps[((size_t)ph * PW + pw) * gh * gw];
                    float acc = 0.f;
                    for (int s = 0; s < gh * gw; ++s) {
                        float val = 0.f;
                        if (t[s].y_low >= 0) {
                            float v1 = plane[t[s].y_low * W + t[s].x_low];
                            float v2 = plane[t[s].y_low * W + t[s].x_high];
                            float v3 = plane[t[s].y_high * W + t[s].x_low];
                            float v4 = plane[t[s].y_high * W + t[s].x_high];
                            if (g_fused)
                                val = fmaf(v4, t[s].w4, fmaf(v3, t[s].w3, fmaf(v1, t[s].w1, v2 * t[s].w2)));
                            else
                                val = ((t[s].w1 * v1 + t[s].w2 * v2) + t[s].w3 * v3) + t[s].w4 * v4;
                        }
                        acc = acc + val;
                    }
                    out[ph * PW + pw] = acc / count;
                }
        }
        free(taps);
    }
}

/* Backward.  The reference scatters with fp32 atomicAdd (order undefined).  This restatement adds
 * the same per-tap terms  g_k = FMUL(top, w_k) / count  in ascending output-index order (the order
 * a serial execution of the reference's CUDA_1D_KERNEL_LOOP would use).  `acc64` != 0 accumulates
 * in double instead (used by the tests to bound the reorder noise). */
ORACLE_API void oracle_roi_align_backward(const float* top_diff, const float* rois, int N, int C, int H, int W,
                                          int R, int PH, int PW, float scale, int sr, float* bottom_diff,
                                          int acc64) {
    size_t total = (size_t)N * C * H * W;
    double* dacc = NULL;
    if (acc64) dacc = (double*)calloc(total, sizeof(double));
    memset(bottom_diff, 0, total * sizeof(float));
    /* parallel over channels: every (n,c) plane is touched by exactly one thread -> deterministic */
#pragma omp parallel for schedule(static)
    for (int c = 0; c < C; ++c) {
        for (int n = 0; n < R; ++n) {
            int b, gh, gw; float sw, sh, bw, bh;
            xfrom_roi_geometry(rois + 5 * n, scale, PH, PW, sr, &b, &sw, &sh, &bw, &bh, &gw, &gh);
            const float count = (float)(gh * gw);
            size_t poff = ((size_t)b * C + c) * H * W;
            const float* tp = top_diff + ((size_t)n * C + c) * PH * PW;
            for (int ph = 0; ph < PH; ++ph)
                for (int pw = 0; pw < PW; ++pw) {
                    float g = tp[ph * PW + pw];
                    for (int iy = 0; iy < gh; ++iy) {
                        float y = xfrom_coord(sh, bh, ph, iy, gh);
                        for (int ix = 0; ix < gw; ++ix) {
                            float x = xfrom_coord(sw, bw, pw, ix, gw);
                            tap_t t; xfrom_taps(H, W, y, x, &t);
                            if (t.x_low < 0) continue;
                            float g1 = (g * t.w1) / count, g2 = (g * t.w2) / count;
                            float g3 = (g * t.w3) / count, g4 = (g * t.w4) / count;
                            size_t i1 = poff + (size_t)t.y_low * W + t.x_low, i2 = poff + (size_t)t.y_low * W + t.x_high;
                            size_t i3 = poff + (size_t)t.y_high * W + t.x_low, i4 = poff + (size_t)t.y_high * W + t.x_high;
                            if (acc64) { dacc[i1] += g1; dacc[i2] += g2; dacc[i3] += g3; dacc[i4] += g4; }
                            else { bottom_diff[i1] += g1; bottom_diff[i2] += g2; bottom_diff[i3] += g3; bottom_diff[i4] += g4; }
                        }
                    }
                }
        }
    }
    if (acc64) {
        for (size_t i = 0; i < total; ++i) bottom_diff[i] = (float)dacc[i];
        free(dacc);
    }
}

/* Number of distinct (n,y,x) feature-map cells hit by any bilinear tap (same for every channel):
 * the "touched_cells" term of the algorithmic-bytes formula in SURVEY.md 8(d). */
ORACLE_API long oracle_roi_align_touched_cells(const float* rois, int N, int H, int W, int R, int PH, int PW,
                                               float scale, int sr) {
    unsigned char* hit = (unsigned char*)calloc((size_t)N * H * W, 1);
    for (int n = 0; n < R; ++n) {
        int b, gh, gw; float sw, sh, bw, bh;
        xfrom_roi_geometry(rois + 5 * n, scale, PH, PW, sr, &b, &sw, &sh, &bw, &bh, &gw, &gh);
        if (b < 0 || b >= N) continue;
        for (int ph = 0; ph < PH; ++ph) for (int iy = 0; iy < gh; ++iy) {
            float y = xfrom_coord(sh, bh, ph, iy, gh);
            for (int pw = 0; pw < PW; ++pw) for (int ix = 0; ix < gw; ++ix) {
                float x = xfrom_coord(sw, bw, pw, ix, gw);
                tap_t t; xfrom_taps(H, W, y, x, &t);
                if (t.x_low < 0) continue;
                unsigned char* p = hit + (size_t)b * H * W;
                p[t.y_low * W + t.x_low] = 1; p[t.y_low * W + t.x_high] = 1;
                p[t.y_high * W + t.x_low] = 1; p[t.y_high * W + t.x_high] = 1;
            }
        }
    }
    long cnt = 0;
    for (size_t i = 0; i < (size_t)N * H * W; ++i) cnt += hit[i];
    free(hit);
    return cnt;
}

/* ------------------------------------------------------------------------------------------
 * RoIAlign, legacy variant
 * reference: lib/model/roi_align/src/roi_align_kernel.cu  ROIAlignForward :15-70, ROIAlignBackward :94-143
 * SASS recipe (sm_100a): the `1.` literals make part of the arithmetic double:
 *   start   = FMUL(x1, scale);  roi_w = FMNMX(0, FADD(FFMA(x2, scale, -start), 1))
 *   bin     = (float)((double)roi_w / (double)(P - 1))
 *   h       = FFMA((float)ph, bin_h, start_h)
 *   hstart  = (int)fminf(floorf(h), H-2);   h_ratio = FADD(h, -(float)hstart)   (float)
 *             taps at rows hstart, hstart + 1 and columns wstart, wstart + 1
 * DEPARTURE from the reference (the only one): on a one-row map (H = 1) the reference's hstart is -1, so it reads
 *   and scatters into row -1, outside the channel plane (W = 1: column -1).  Here, as in roi_align_legacy.cu,
 *   hstart = max(min(floor(h), H-2), 0) and the second tap row is min(hstart + 1, H - 1) (same for columns), so on a
 *   one-row map both taps are row 0; the weights are unchanged.  For H, W >= 2 this is the reference's arithmetic.
 *   fwd     = (float)( DADD( DFMA(omw, (double)FMUL(hr, dl),
 *                               DFMA(DMUL((double)ul, omh), omw, DMUL((double)wr, DMUL(omh,(double)ur)))),
 *                            (double)FMUL(wr, FMUL(hr, dr)) ) )
 *             with omh = 1.0 - (double)hr, omw = 1.0 - (double)wr
 *   bwd     : ul += (float)(((double)g*omh) * (double)(1.f - wr)),  ur += (float)(((double)g*omh)*(double)wr),
 *             dl += (1.f - wr) * (hr * g),  dr += wr * (hr * g)
 * ------------------------------------------------------------------------------------------ */
static inline int legacy_geometry(const float* roi, float scale, int PH, int PW, int H, int W, int ph, int pw,
                                  float* h_ratio, float* w_ratio, int* hstart, int* wstart, int* dh, int* dw) {
    float sw = roi[1] * scale, sh = roi[2] * scale;
    float rw = fmaxf(fmaf(roi[3], scale, -sw) + 1.f, 0.f);
    float rh = fmaxf(fmaf(roi[4], scale, -sh) + 1.f, 0.f);
    float bh = (float)((double)rh / ((double)PH - 1.));
    float bw = (float)((double)rw / ((double)PW - 1.));
    float h = fmaf((float)ph, bh, sh);
    float w = fmaf((float)pw, bw, sw);
    *hstart = (int)fmaxf(fminf(floorf(h), (float)(H - 2)), 0.f);
    *wstart = (int)fmaxf(fminf(floorf(w), (float)(W - 2)), 0.f);
    *dh = (*hstart + 1 <= H - 1) ? W : 0;     /* offset of the lower taps from the upper ones */
    *dw = (*wstart + 1 <= W - 1) ? 1 : 0;
    if (h < 0 || h >= (float)H || w < 0 || w >= (float)W) return 0;
    *h_ratio = h - (float)(*hstart);
    *w_ratio = w - (float)(*wstart);
    return 1;
}

ORACLE_API void oracle_roi_align_legacy_forward(const float* bottom, const float* rois, int N, int C, int H, int W,
                                                int R, int PH, int PW, float scale, float* top) {
    (void)N;
#pragma omp parallel for schedule(dynamic, 1)
    for (int n = 0; n < R; ++n) {
        /* the reference keeps the batch index as a float and multiplies: (int)(b * C * H * W) */
        int img_start = (int)(rois[5 * n] * (float)C * (float)H * (float)W);
        for (int c = 0; c < C; ++c)
            for (int ph = 0; ph < PH; ++ph)
                for (int pw = 0; pw < PW; ++pw) {
                    float hr, wr; int hs, ws, dh, dw;
                    float* o = top + (((size_t)n * C + c) * PH + ph) * PW + pw;
                    if (!legacy_geometry(rois + 5 * n, scale, PH, PW, H, W, ph, pw, &hr, &wr, &hs, &ws, &dh, &dw)) { *o = 0.f; continue; }
                    const float* p = bottom + img_start + ((size_t)c * H + hs) * W + ws;
                    float ul = p[0], ur = p[dw], dl = p[dh], dr = p[dh + dw];
                    double omh = 1.0 - (double)hr, omw = 1.0 - (double)wr;
                    double t_ur = (double)wr * (omh * (double)ur);
                    double acc = fma((double)ul * omh, omw, t_ur);
                    acc = fma(omw, (double)(hr * dl), acc);
                    acc = acc + (double)(wr * (hr * dr));
                    *o = (float)acc;
                }
    }
}

ORACLE_API void oracle_roi_align_legacy_backward(const float* top_diff, const float* rois, int N, int C, int H, int W,
                                                 int R, int PH, int PW, float scale, float* bottom_diff, int acc64) {
    size_t total = (size_t)N * C * H * W;
    double* dacc = acc64 ? (double*)calloc(total, sizeof(double)) : NULL;
    memset(bottom_diff, 0, total * sizeof(float));
#pragma omp parallel for schedule(static)
    for (int c = 0; c < C; ++c)
        for (int n = 0; n < R; ++n) {
            int img_start = (int)(rois[5 * n] * (float)C * (float)H * (float)W);
            for (int ph = 0; ph < PH; ++ph)
                for (int pw = 0; pw < PW; ++pw) {
                    float hr, wr; int hs, ws, dh, dw;
                    if (!legacy_geometry(rois + 5 * n, scale, PH, PW, H, W, ph, pw, &hr, &wr, &hs, &ws, &dh, &dw)) continue;
                    float g = top_diff[(((size_t)n * C + c) * PH + ph) * PW + pw];
                    size_t ul = (size_t)img_start + ((size_t)c * H + hs) * W + ws;
                    double gomh = (double)g * (1.0 - (double)hr);
                    float omw = 1.f - wr;
                    float g_ul = (float)(gomh * (double)omw);
                    float g_ur = (float)(gomh * (double)wr);
                    float ghr = hr * g;
                    float g_dl = omw * ghr;
                    float g_dr = wr * ghr;
                    if (acc64) { dacc[ul] += g_ul; dacc[ul + dw] += g_ur; dacc[ul + dh] += g_dl; dacc[ul + dh + dw] += g_dr; }
                    else { bottom_diff[ul] += g_ul; bottom_diff[ul + dw] += g_ur; bottom_diff[ul + dh] += g_dl; bottom_diff[ul + dh + dw] += g_dr; }
                }
        }
    if (acc64) { for (size_t i = 0; i < total; ++i) bottom_diff[i] = (float)dacc[i]; free(dacc); }
}

/* ------------------------------------------------------------------------------------------
 * RoIPool
 * reference: lib/model/roi_pooling/src/roi_pooling_kernel.cu  ROIPoolForward :24-93, ROIPoolBackward :128-203
 * (the CUDA kernels, NOT the buggy CPU file src/roi_pooling.c -- SURVEY.md 2.2)
 *   roi_start = (int)roundf(FMUL(x, scale));  roi_w = max(end - start + 1, 1)
 *   bin = (float)roi_w / (float)P;  hstart = (int)floorf((float)ph * bin) ... clipped to [0, H]
 *   strict '>' max, first maximum wins, argmax = flat index into the WHOLE bottom tensor (int32)
 * ------------------------------------------------------------------------------------------ */
ORACLE_API void oracle_roi_pool_forward(const float* bottom, const float* rois, int N, int C, int H, int W,
                                        int R, int PH, int PW, float scale, float* top, int* argmax) {
    (void)N;
#pragma omp parallel for schedule(dynamic, 1)
    for (int n = 0; n < R; ++n) {
        const float* roi = rois + 5 * n;
        int b = (int)roi[0];
        int rsw = (int)roundf(roi[1] * scale), rsh = (int)roundf(roi[2] * scale);
        int rew = (int)roundf(roi[3] * scale), reh = (int)roundf(roi[4] * scale);
        int rw = (int)fmaxf((float)(rew - rsw + 1), 1.f), rh = (int)fmaxf((float)(reh - rsh + 1), 1.f);
        float bh = (float)rh / (float)PH, bw = (float)rw / (float)PW;
        for (int c = 0; c < C; ++c) {
            int off = (b * C + c) * H * W;
            for (int ph = 0; ph < PH; ++ph)
                for (int pw = 0; pw < PW; ++pw) {
                    int hs = (int)floorf((float)ph * bh), ws = (int)floorf((float)pw * bw);
                    int he = (int)ceilf((float)(ph + 1) * bh), we = (int)ceilf((float)(pw + 1) * bw);
                    hs = (int)fminf(fmaxf((float)(hs + rsh), 0.f), (float)H);
                    he = (int)fminf(fmaxf((float)(he + rsh), 0.f), (float)H);
                    ws = (int)fminf(fmaxf((float)(ws + rsw), 0.f), (float)W);
                    we = (int)fminf(fmaxf((float)(we + rsw), 0.f), (float)W);
                    int empty = (he <= hs) || (we <= ws);
                    float maxval = empty ? 0.f : -FLT_MAX;
                    int maxidx = -1;
                    for (int h = hs; h < he; ++h)
                        for (int w = ws; w < we; ++w) {
                            float v = bottom[off + h * W + w];
                            if (v > maxval) { maxval = v; maxidx = off + h * W + w; }
                        }
                    size_t o = (((size_t)n * C + c) * PH + ph) * PW + pw;
                    top[o] = maxval;
                    if (argmax) argmax[o] = maxidx;
                }
        }
    }
}

/* Per-input-cell gather in the reference's own loop order (RoIs ascending, then ph, pw) so the
 * fp32 sum is bit-identical to the (deterministic) reference kernel. */
ORACLE_API void oracle_roi_pool_backward(const float* top_diff, const int* argmax, const float* rois,
                                         int N, int C, int H, int W, int R, int PH, int PW, float scale,
                                         float* bottom_diff) {
#pragma omp parallel for schedule(static) collapse(2)
    for (int n = 0; n < N; ++n)
        for (int c = 0; c < C; ++c)
            for (int h = 0; h < H; ++h)
                for (int w = 0; w < W; ++w) {
                    int index = ((n * C + c) * H + h) * W + w;
                    float grad = 0.f;
                    for (int r = 0; r < R; ++r) {
                        const float* roi = rois + 5 * r;
                        if (n != (int)roi[0]) continue;
                        int rsw = (int)roundf(roi[1] * scale), rsh = (int)roundf(roi[2] * scale);
                        int rew = (int)roundf(roi[3] * scale), reh = (int)roundf(roi[4] * scale);
                        if (!(w >= rsw && w <= rew && h >= rsh && h <= reh)) continue;
                        int rw = (int)fmaxf((float)(rew - rsw + 1), 1.f), rh = (int)fmaxf((float)(reh - rsh + 1), 1.f);
                        float bh = (float)rh / (float)PH, bw = (float)rw / (float)PW;
                        int phs = (int)floorf((float)(h - rsh) / bh), phe = (int)ceilf((float)(h - rsh + 1) / bh);
                        int pws = (int)floorf((float)(w - rsw) / bw), pwe = (int)ceilf((float)(w - rsw + 1) / bw);
                        phs = (int)fminf(fmaxf((float)phs, 0.f), (float)PH); phe = (int)fminf(fmaxf((float)phe, 0.f), (float)PH);
                        pws = (int)fminf(fmaxf((float)pws, 0.f), (float)PW); pwe = (int)fminf(fmaxf((float)pwe, 0.f), (float)PW);
                        size_t off = (size_t)r * C * PH * PW;
                        for (int ph = phs; ph < phe; ++ph)
                            for (int pw = pws; pw < pwe; ++pw) {
                                size_t o = off + ((size_t)c * PH + ph) * PW + pw;
                                if (argmax[o] == index) grad += top_diff[o];
                            }
                    }
                    bottom_diff[index] = grad;
                }
}

/* ------------------------------------------------------------------------------------------
 * RoICrop (bilinear sampler from an explicit (y,x) grid), dense NCHW image, (R,h,w,2) grid
 * reference: lib/model/roi_crop/src/roi_crop_cuda_kernel.cu
 *   getTopLeft :11-22, bilinearSamplingFromGrid :47-109, backwardBilinearSampling :111-194
 * SASS recipe: coord = FMUL.D2(FADD(g,1), (float)(size-1));  point = floor(coord);
 *   weight = FADD(FADD(point, -coord), 1)
 *   v = FFMA(FMUL(1-xW,1-yW), BR, FFMA(FMUL(xW,1-yW), BL, FFMA(FMUL(xW,yW), TL, FMUL(FMUL(yW,1-xW), TR))))
 *   bwd: gradImg[tap] += FMUL(g, FMUL(wa, wb));  the CUDA kernel never writes the grid gradient.
 * Image index of RoI b is b / (R / N)  (:64, :217).
 * ------------------------------------------------------------------------------------------ */
static inline void crop_topleft(float g, int size, int* point, float* weight) {
    float coord = ((g + 1.f) * (float)(size - 1)) * 0.5f;
    float fl = floorf(coord);
    *point = (int)fl;
    *weight = (fl - coord) + 1.f;
}

ORACLE_API void oracle_roi_crop_forward(const float* img, const float* grid, int N, int C, int H, int W,
                                        int R, int oh, int ow, float* out) {
    int per = R / N;
    memset(out, 0, sizeof(float) * (size_t)R * C * oh * ow);
#pragma omp parallel for schedule(static)
    for (int b = 0; b < R; ++b) {
        int bi = b / per;
        for (int y = 0; y < oh; ++y)
            for (int x = 0; x < ow; ++x) {
                const float* g = grid + (((size_t)b * oh + y) * ow + x) * 2;
                int yt, xl; float yW, xW;
                crop_topleft(g[1], W, &xl, &xW);
                crop_topleft(g[0], H, &yt, &yW);
                int xin0 = xl >= 0 && xl <= W - 1, xin1 = xl + 1 >= 0 && xl + 1 <= W - 1;
                int yin0 = yt >= 0 && yt <= H - 1, yin1 = yt + 1 >= 0 && yt + 1 <= H - 1;
                int tl = xin0 && yin0, tr = xin1 && yin0, bl = xin0 && yin1, br = xin1 && yin1;
                if (!tl && !tr && !bl && !br) continue;
                float omx = 1.f - xW, omy = 1.f - yW;
                float w_tr = yW * omx, w_tl = xW * yW, w_bl = xW * omy, w_br = omx * omy;
                for (int c = 0; c < C; ++c) {
                    const float* p = img + ((size_t)bi * C + c) * H * W + (ptrdiff_t)yt * W + xl;
                    float vtl = tl ? p[0] : 0.f, vtr = tr ? p[1] : 0.f, vbl = bl ? p[W] : 0.f, vbr = br ? p[W + 1] : 0.f;
                    float v = fmaf(w_br, vbr, fmaf(w_bl, vbl, fmaf(w_tl, vtl, w_tr * vtr)));
                    out[(((size_t)b * C + c) * oh + y) * ow + x] = v;
                }
            }
    }
}

ORACLE_API void oracle_roi_crop_backward(const float* grad_out, const float* grid, int N, int C, int H, int W,
                                         int R, int oh, int ow, float* grad_img, int acc64) {
    int per = R / N;
    size_t total = (size_t)N * C * H * W;
    double* dacc = acc64 ? (double*)calloc(total, sizeof(double)) : NULL;
    memset(grad_img, 0, total * sizeof(float));
#pragma omp parallel for schedule(static)
    for (int c = 0; c < C; ++c)
        for (int b = 0; b < R; ++b) {
            int bi = b / per;
            for (int y = 0; y < oh; ++y)
                for (int x = 0; x < ow; ++x) {
                    const float* g = grid + (((size_t)b * oh + y) * ow + x) * 2;
                    int yt, xl; float yW, xW;
                    crop_topleft(g[1], W, &xl, &xW);
                    crop_topleft(g[0], H, &yt, &yW);
                    int xin0 = xl >= 0 && xl <= W - 1, xin1 = xl + 1 >= 0 && xl + 1 <= W - 1;
                    int yin0 = yt >= 0 && yt <= H - 1, yin1 = yt + 1 >= 0 && yt + 1 <= H - 1;
                    float go = grad_out[(((size_t)b * C + c) * oh + y) * ow + x];
                    float omx = 1.f - xW, omy = 1.f - yW;
                    ptrdiff_t base = (ptrdiff_t)(((size_t)bi * C + c) * H * W) + (ptrdiff_t)yt * W + xl;
                    float gtl = go * (xW * yW), gtr = go * (omx * yW), gbl = go * (xW * omy), gbr = go * (omx * omy);
                    if (acc64) {
                        if (xin0 && yin0) dacc[base] += gtl;
                        if (xin1 && yin0) dacc[base + 1] += gtr;
                        if (xin0 && yin1) dacc[base + W] += gbl;
                        if (xin1 && yin1) dacc[base + W + 1] += gbr;
                    } else {
                        if (xin0 && yin0) grad_img[base] += gtl;
                        if (xin1 && yin0) grad_img[base + 1] += gtr;
                        if (xin0 && yin1) grad_img[base + W] += gbl;
                        if (xin1 && yin1) grad_img[base + W + 1] += gbr;
                    }
                }
        }
    if (acc64) { for (size_t i = 0; i < total; ++i) grad_img[i] = (float)dacc[i]; free(dacc); }
}

/* ------------------------------------------------------------------------------------------
 * NMS, CUDA semantics (bit-exact target)
 * reference: lib/model/nms/src/nms_cuda_kernel.cu  devIoU :31-39, nms_kernel :41-85, host scan :123-144
 * SASS recipe (a = row box = lower index, b = column box = higher index):
 *   Sa    = FMUL(FADD(FADD(a2,-a0),1), FADD(FADD(a3,-a1),1))
 *   w     = FMNMX(0, FADD(FADD(min(a2,b2), -max(a0,b0)), 1));  h likewise;  inter = FMUL(w,h)
 *   den   = FADD(FFMA(FADD(FADD(b2,-b0),1), FADD(FADD(b3,-b1),1), Sa), -inter)
 *   bit   = (inter / den) > thresh          (IEEE RN division; NaN compares false)
 * Greedy scan: box j is removed iff some kept i < j has bit(i,j).  Boxes are assumed sorted by the
 * caller (the function never sorts and never reads column 4).  keep_out: ascending kept indices.
 * ------------------------------------------------------------------------------------------ */
static inline int nms_cuda_bit(const float* a, const float* b, float thresh) {
    float Sa = ((a[2] - a[0]) + 1.f) * ((a[3] - a[1]) + 1.f);
    float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
    float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
    float w = fmaxf((right - left) + 1.f, 0.f), h = fmaxf((bottom - top) + 1.f, 0.f);
    float inter = w * h;
    float t = fmaf((b[2] - b[0]) + 1.f, (b[3] - b[1]) + 1.f, Sa);
    float den = t - inter;
    return (inter / den) > thresh;
}

ORACLE_API int oracle_nms_cuda(const float* boxes, int n, int dim, float thresh, int* keep_out) {
    unsigned char* removed = (unsigned char*)calloc((size_t)(n > 0 ? n : 1), 1);
    int kept = 0;
    for (int i = 0; i < n; ++i) {
        if (removed[i]) continue;
        keep_out[kept++] = i;
        const float* a = boxes + (size_t)i * dim;
#pragma omp parallel for schedule(static) if (n - i > 4096)
        for (int j = i + 1; j < n; ++j)
            if (!removed[j] && nms_cuda_bit(a, boxes + (size_t)j * dim, thresh)) removed[j] = 1;
    }
    free(removed);
    return kept;
}

/* The 64-bit suppression mask exactly as nms_kernel writes it (incl. lower-triangle blocks and
 * the diagonal-block rule `start = t + 1`), for checking the device mask word for word. */
ORACLE_API void oracle_nms_cuda_mask(const float* boxes, int n, int dim, float thresh, uint64_t* mask) {
    int cb = (n + 63) / 64;
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i)
        for (int cbk = 0; cbk < cb; ++cbk) {
            uint64_t t = 0;
            int col_size = n - cbk * 64 < 64 ? n - cbk * 64 : 64;
            int start = (i / 64 == cbk) ? (i % 64) + 1 : 0;
            for (int k = start; k < col_size; ++k)
                if (nms_cuda_bit(boxes + (size_t)i * dim, boxes + (size_t)(cbk * 64 + k) * dim, thresh)) t |= 1ULL << k;
            mask[(size_t)i * cb + cbk] = t;
        }
}

/* ------------------------------------------------------------------------------------------
 * NMS, the reference's LIVE CPU flavour (secondary oracle; NOT the bit-exact target)
 * reference: lib/utils/cython_nms.pyx:37-87 -- sorts by score internally, rounded per-box areas,
 * unfused IoU, suppress on `>=`, returns ascending ORIGINAL indices of the survivors.
 * ------------------------------------------------------------------------------------------ */
typedef struct { float s; int i; } si_t;
static int si_cmp(const void* a, const void* b) {
    const si_t* x = (const si_t*)a; const si_t* y = (const si_t*)b;
    if (x->s > y->s) return -1;
    if (x->s < y->s) return 1;
    return (x->i < y->i) ? 1 : -1;   /* numpy argsort()[::-1]: ties come out in descending index */
}
ORACLE_API int oracle_nms_cython(const float* dets, int n, double thresh, int* keep_out) {
    si_t* order = (si_t*)malloc(sizeof(si_t) * (size_t)(n > 0 ? n : 1));
    float* areas = (float*)malloc(sizeof(float) * (size_t)(n > 0 ? n : 1));
    unsigned char* sup = (unsigned char*)calloc((size_t)(n > 0 ? n : 1), 1);
    for (int i = 0; i < n; ++i) {
        const float* d = dets + 5 * (size_t)i;
        order[i].s = d[4]; order[i].i = i;
        areas[i] = (d[2] - d[0] + 1.f) * (d[3] - d[1] + 1.f);
    }
    qsort(order, (size_t)n, sizeof(si_t), si_cmp);
    for (int _i = 0; _i < n; ++_i) {
        int i = order[_i].i;
        if (sup[i]) continue;
        const float* a = dets + 5 * (size_t)i;
        for (int _j = _i + 1; _j < n; ++_j) {
            int j = order[_j].i;
            if (sup[j]) continue;
            const float* b = dets + 5 * (size_t)j;
            float xx1 = fmaxf(a[0], b[0]), yy1 = fmaxf(a[1], b[1]);
            float xx2 = fminf(a[2], b[2]), yy2 = fminf(a[3], b[3]);
            float w = fmaxf(0.f, xx2 - xx1 + 1.f), h = fmaxf(0.f, yy2 - yy1 + 1.f);
            float inter = w * h;
            float ovr = inter / (areas[i] + areas[j] - inter);
            if ((double)ovr >= thresh) sup[j] = 1;   /* thresh is a Python float (double) in the .pyx */
        }
    }
    int kept = 0;
    for (int i = 0; i < n; ++i) if (!sup[i]) keep_out[kept++] = i;
    free(order); free(areas); free(sup);
    return kept;
}
