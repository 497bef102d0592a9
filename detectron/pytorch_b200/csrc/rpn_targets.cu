// rpn_targets.cu -- RPN anchor labels and box-regression targets on the device (the training-time add_rpn_blobs).
//
// The reference does this on the host, per image, in numpy + Cython, before every training step:
//   lib/roi_data/data_utils.py:50-101     get_field_of_anchors: cell anchors + integer shifts in float64, cast to float32
//   lib/roi_data/rpn.py:115-134           inside test against the image (RPN_STRADDLE_THRESH; < 0 keeps every anchor)
//   lib/roi_data/rpn.py:140-170           IoU matrix (cython_bbox.bbox_overlaps), per-anchor max / argmax, per-gt max over the
//                                         inside anchors, fg = ties of a column max or row max >= RPN_POSITIVE_OVERLAP
//   lib/roi_data/rpn.py:172-190           fg subsample (npr.choice without replacement), bg candidates (row max < NEGATIVE,
//                                         fg included), bg draw with replacement (npr.randint) applied only when there are
//                                         more candidates than the minibatch needs
//   lib/roi_data/rpn.py:192-261           targets for the fg set as it stood BEFORE the bg draw, weights, unmap, and the
//                                         (1, A, F, F) / (1, 4A, F, F) split per field of anchors
// All images and all levels of a call go through the same launches:
//   labelling half  memset + colmax + label + compact            (3 kernels; the fg / bg candidate counts are the one host read)
//   emit half       scatter draw + count examples + emit blobs    (3 kernels)
// Anchors are recomputed wherever they are needed; no field-of-anchors table is kept.
#include "common.cuh"

namespace b200 {

constexpr int kRpnMaxLevels = 8;
constexpr int kRpnMaxCellAnchors = 32;
constexpr int kRpnMaxImages = 64;

namespace {

constexpr int kRpnTile = 1024;       // anchors per CTA in the label / compact kernels (256 threads x 4)

// flag bits, one byte per (image, anchor)
constexpr unsigned kInside = 1u, kFgCand = 2u, kBgCand = 4u, kDisabled = 8u, kEnabled = 16u;

struct RpnGeom {
    int num_levels, num_images, total;          // total: anchors per image, all levels
    int F[kRpnMaxLevels], A[kRpnMaxLevels], cell0[kRpnMaxLevels];
    int start[kRpnMaxLevels + 1];               // first anchor of each level in the reference's concatenated order
    double stride[kRpnMaxLevels];
    double cell[kRpnMaxCellAnchors][4];         // generate_anchors output, float64 as the reference keeps it
    double xmax[kRpnMaxImages], ymax[kRpnMaxImages];   // im_w + straddle, im_h + straddle (float64 comparison)
    float xymin;                                // float32(-straddle)
    int keep_all;                               // straddle < 0
    int gt_begin[kRpnMaxImages + 1];
};

struct RpnDraws {
    int dis_begin[kRpnMaxImages + 1], en_begin[kRpnMaxImages + 1];
};

struct RpnOut {
    int* labels[kRpnMaxLevels];
    float* targets[kRpnMaxLevels];
    float* inside[kRpnMaxLevels];
    float* outside[kRpnMaxLevels];
    int unit_start[kRpnMaxLevels + 1];          // per level A * ceil(F * F / 4) work units of four plane positions
};

__device__ __forceinline__ int rpn_level(const RpnGeom& g, int idx) {
    int l = 0;
    while (l + 1 < g.num_levels && idx >= g.start[l + 1]) ++l;
    return l;
}

// anchor `idx` (level-major, then (h, w, a)): float32(float64(cell anchor) + float64(shift)), data_utils.py:69-93
__device__ __forceinline__ float4 rpn_anchor(const RpnGeom& g, int l, int idx) {
    const int local = idx - g.start[l], A = g.A[l], F = g.F[l];
    const int a = local % A, cellidx = local / A;
    const double sx = __dmul_rn((double)(cellidx % F), g.stride[l]), sy = __dmul_rn((double)(cellidx / F), g.stride[l]);
    const double* c = g.cell[g.cell0[l] + a];
    return make_float4((float)__dadd_rn(c[0], sx), (float)__dadd_rn(c[1], sy), (float)__dadd_rn(c[2], sx), (float)__dadd_rn(c[3], sy));
}

__device__ __forceinline__ bool rpn_inside(const RpnGeom& g, int n, float4 b) {
    return g.keep_all || (b.x >= g.xymin && b.y >= g.xymin && (double)b.z < g.xmax[n] && (double)b.w < g.ymax[n]);
}

__device__ __forceinline__ float rpn_iou(float4 b, float4 q, float qarea) { return cython_iou(b.x, b.y, b.z, b.w, q.x, q.y, q.z, q.w, qarea); }

// pass 1: per ground-truth box, the maximum IoU over the inside anchors (rpn.py:154-159).  IoU >= 0, so a max on the float
// bits is exact and independent of the order of the atomics.
__global__ void __launch_bounds__(256)
rpn_colmax_kernel(const __grid_constant__ RpnGeom g, const float4* __restrict__ gt, unsigned* __restrict__ colmax) {
    __shared__ float4 s_gt[256];
    __shared__ float s_area[256];
    __shared__ unsigned s_max[256];
    const int n = blockIdx.y, idx = blockIdx.x * 256 + threadIdx.x;
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    bool in = false;
    if (idx < g.total) {
        b = rpn_anchor(g, rpn_level(g, idx), idx);
        in = rpn_inside(g, n, b);
    }
    const int g0 = g.gt_begin[n], G = g.gt_begin[n + 1] - g0;
    for (int c0 = 0; c0 < G; c0 += 256) {
        __syncthreads();
        if (c0 + (int)threadIdx.x < G) {
            const float4 q = __ldg(gt + g0 + c0 + threadIdx.x);
            s_gt[threadIdx.x] = q; s_area[threadIdx.x] = cython_area(q.x, q.y, q.z, q.w); s_max[threadIdx.x] = 0u;
        }
        __syncthreads();
        const int m = min(256, G - c0);
        if (in) {
            for (int j = 0; j < m; ++j) {
                const unsigned u = __float_as_uint(rpn_iou(b, s_gt[j], s_area[j]));
                if (u > s_max[j]) atomicMax(s_max + j, u);
            }
        }
        __syncthreads();
        if ((int)threadIdx.x < m && s_max[threadIdx.x] != 0u) atomicMax(colmax + g0 + c0 + threadIdx.x, s_max[threadIdx.x]);
    }
}

// pass 2: the row again -- first maximum (np.argmax), exact ties with a column maximum (rpn.py:160-170), fg / bg candidates.
// Writes the flag byte of every anchor, the argmax of the fg candidates and the CTA's (fg, bg, inside) counts.
__global__ void __launch_bounds__(256)
rpn_label_kernel(const __grid_constant__ RpnGeom g, const float4* __restrict__ gt, const unsigned* __restrict__ colmax, float pos_thresh,
                 float neg_thresh, long long tpad, unsigned char* __restrict__ flags, int* __restrict__ argmax, int* __restrict__ blk_counts) {
    __shared__ float4 s_gt[256];
    __shared__ float s_area[256], s_cmax[256];
    __shared__ int s_cnt[3];
    const int n = blockIdx.y, t = threadIdx.x;
    if (t < 3) s_cnt[t] = 0;
    float4 b[4];
    bool in[4], tie[4];
    float best[4];
    int arg[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int idx = blockIdx.x * kRpnTile + k * 256 + t;
        in[k] = false; tie[k] = false; best[k] = -1.f; arg[k] = 0;
        b[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (idx < g.total) {
            b[k] = rpn_anchor(g, rpn_level(g, idx), idx);
            in[k] = rpn_inside(g, n, b[k]);
        }
    }
    const int g0 = g.gt_begin[n], G = g.gt_begin[n + 1] - g0;
    for (int c0 = 0; c0 < G; c0 += 256) {
        __syncthreads();
        if (c0 + t < G) {
            const float4 q = __ldg(gt + g0 + c0 + t);
            s_gt[t] = q; s_area[t] = cython_area(q.x, q.y, q.z, q.w); s_cmax[t] = __uint_as_float(__ldg(colmax + g0 + c0 + t));
        }
        __syncthreads();
        const int m = min(256, G - c0);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if (!in[k]) continue;
            for (int j = 0; j < m; ++j) {
                const float o = rpn_iou(b[k], s_gt[j], s_area[j]);
                if (o > best[k]) { best[k] = o; arg[k] = c0 + j; }            // strict >: the first maximum wins
                tie[k] |= (o == s_cmax[j]);
            }
        }
    }
    const int lane = t & 31;
    int cf = 0, cb = 0, ci = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int idx = blockIdx.x * kRpnTile + k * 256 + t;
        const bool fg = in[k] && (tie[k] || best[k] >= pos_thresh);
        const bool bg = in[k] && best[k] < neg_thresh;
        if (idx < g.total) {
            flags[n * tpad + idx] = (unsigned char)((in[k] ? kInside : 0u) | (fg ? kFgCand : 0u) | (bg ? kBgCand : 0u));
            if (fg) argmax[(long long)n * g.total + idx] = arg[k];
        }
        cf += __popc(__ballot_sync(0xffffffffu, fg));
        cb += __popc(__ballot_sync(0xffffffffu, bg));
        ci += __popc(__ballot_sync(0xffffffffu, in[k]));
    }
    if (lane == 0) { atomicAdd(s_cnt, cf); atomicAdd(s_cnt + 1, cb); atomicAdd(s_cnt + 2, ci); }
    __syncthreads();
    if (t < 3) blk_counts[((long long)n * gridDim.x + blockIdx.x) * 3 + t] = s_cnt[t];
}

// pass 3: ascending index lists of the fg and bg candidates per image (np.where order); the last CTA of each image writes
// the image's (fg, bg, inside) counts.
__global__ void __launch_bounds__(256)
rpn_compact_kernel(int total, long long tpad, const unsigned char* __restrict__ flags, const int* __restrict__ blk_counts,
                   int* __restrict__ fg_list, int* __restrict__ bg_list, int* __restrict__ counts) {
    __shared__ int s_red[3][8];
    __shared__ int s_wf[8], s_wb[8];
    __shared__ int s_base[3];
    const int n = blockIdx.y, blk = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int* bc = blk_counts + (long long)n * gridDim.x * 3;
    int sf = 0, sb = 0, si = 0;
    for (int q = t; q < blk; q += 256) { sf += bc[3 * q]; sb += bc[3 * q + 1]; si += bc[3 * q + 2]; }
    for (int o = 16; o > 0; o >>= 1) {
        sf += __shfl_xor_sync(0xffffffffu, sf, o); sb += __shfl_xor_sync(0xffffffffu, sb, o); si += __shfl_xor_sync(0xffffffffu, si, o);
    }
    if (lane == 0) { s_red[0][warp] = sf; s_red[1][warp] = sb; s_red[2][warp] = si; }
    __syncthreads();
    if (t < 3) {
        int s = 0;
        for (int w = 0; w < 8; ++w) s += s_red[t][w];
        s_base[t] = s;
    }
    __syncthreads();
    int pf = s_base[0], pb = s_base[1];
    int* fl = fg_list + (long long)n * total;
    int* bl = bg_list + (long long)n * total;
    for (int k = 0; k < 4; ++k) {
        const int idx = blk * kRpnTile + k * 256 + t;
        const unsigned f8 = idx < total ? flags[n * tpad + idx] : 0u;
        const bool f = f8 & kFgCand, b = f8 & kBgCand;
        const unsigned mf = __ballot_sync(0xffffffffu, f), mb = __ballot_sync(0xffffffffu, b);
        __syncthreads();                                                  // s_wf / s_wb of the previous round are consumed
        if (lane == 0) { s_wf[warp] = __popc(mf); s_wb[warp] = __popc(mb); }
        __syncthreads();
        int of = pf, ob = pb;
        for (int w = 0; w < warp; ++w) { of += s_wf[w]; ob += s_wb[w]; }
        if (f) fl[of + __popc(mf & ((1u << lane) - 1u))] = idx;
        if (b) bl[ob + __popc(mb & ((1u << lane) - 1u))] = idx;
        for (int w = 0; w < 8; ++w) { pf += s_wf[w]; pb += s_wb[w]; }
    }
    if (blk == (int)gridDim.x - 1 && t < 3) {
        const int* own = bc + 3 * blk;
        counts[3 * n + t] = s_base[t] + own[t];
    }
}

// the caller's draw: fg positions disabled (rpn.py:176-179), bg positions enabled (:187-189).  Positions out of range are
// ignored (the host layer validates them).
__global__ void __launch_bounds__(256)
rpn_scatter_draw_kernel(const __grid_constant__ RpnDraws d, int total, long long tpad, const int* __restrict__ counts,
                        const int* __restrict__ fg_disable, const int* __restrict__ bg_enable, const int* __restrict__ fg_list,
                        const int* __restrict__ bg_list, unsigned char* __restrict__ flags) {
    const int n = blockIdx.y, j = blockIdx.x * 256 + threadIdx.x;
    const int nd = d.dis_begin[n + 1] - d.dis_begin[n], ne = d.en_begin[n + 1] - d.en_begin[n];
    int a = -1;
    unsigned bit = 0u;
    if (j < nd) {
        const int p = __ldg(fg_disable + d.dis_begin[n] + j);
        if (p >= 0 && p < __ldg(counts + 3 * n)) { a = __ldg(fg_list + (long long)n * total + p); bit = kDisabled; }
    } else if (j < nd + ne) {
        const int p = __ldg(bg_enable + d.en_begin[n] + (j - nd));
        if (p >= 0 && p < __ldg(counts + 3 * n + 1)) { a = __ldg(bg_list + (long long)n * total + p); bit = kEnabled; }
    }
    if (a < 0) return;
    unsigned char* base = flags + n * tpad;
    atomicOr(reinterpret_cast<unsigned*>(base + (a & ~3)), bit << (8 * (a & 3)));
}

// num_examples = #(labels >= 0) after the draw (rpn.py:212): the fg left by the disable draw, plus every distinct enabled
// anchor that is not one of them.
__global__ void __launch_bounds__(256)
rpn_count_kernel(const __grid_constant__ RpnDraws d, int total, long long tpad, const int* __restrict__ counts,
                 const int* __restrict__ bg_enable, const int* __restrict__ bg_list, const unsigned char* __restrict__ flags,
                 int* __restrict__ num_examples) {
    __shared__ int s_cnt;
    const int n = blockIdx.x, t = threadIdx.x;
    if (t == 0) s_cnt = 0;
    __syncthreads();
    const int nb = __ldg(counts + 3 * n + 1);
    const int* en = bg_enable + d.en_begin[n];
    const int ne = d.en_begin[n + 1] - d.en_begin[n];
    int c = 0;
    for (int j = t; j < ne; j += 256) {
        const int p = __ldg(en + j);
        if (p < 0 || p >= nb) continue;
        bool first = true;
        for (int k = 0; k < j && first; ++k) first = __ldg(en + k) != p;
        if (!first) continue;
        const unsigned f = flags[n * tpad + __ldg(bg_list + (long long)n * total + p)];
        if (!((f & kFgCand) && !(f & kDisabled))) ++c;
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((t & 31) == 0) atomicAdd(&s_cnt, c);
    __syncthreads();
    if (t == 0) {
        const int active = max(__ldg(counts + 3 * n) - (d.dis_begin[n + 1] - d.dis_begin[n]), 0);
        num_examples[n] = active + s_cnt;
    }
}

// the four blobs of every level, every element, in (N, A, F, F) / (N, 4A, F, F) layout (rpn.py:192-259, unmap included).
// One thread = one cell anchor a at four consecutive plane positions; VEC: F * F % 4 == 0, so 16-byte stores.
template <bool VEC>
__device__ __forceinline__ void rpn_emit_unit(const RpnGeom& g, const RpnOut& o, int n, int l, int a, int p0, const float4* __restrict__ gt,
                                              const unsigned char* __restrict__ fl, const int* __restrict__ am, float ow) {
    const int F2 = g.F[l] * g.F[l], A = g.A[l];
    int lab[4];
    float tg[4][4], iw[4], owt[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        lab[i] = -1; iw[i] = 0.f; owt[i] = 0.f;
        tg[0][i] = tg[1][i] = tg[2][i] = tg[3][i] = 0.f;
        const int p = p0 + i;
        if (p >= F2) continue;
        const int idx = g.start[l] + p * A + a;
        const unsigned f = fl[idx];
        const bool fg = (f & kFgCand) && !(f & kDisabled);
        lab[i] = !(f & kInside) ? -1 : (f & kEnabled) ? 0 : fg ? 1 : -1;
        iw[i] = lab[i] == 1 ? 1.f : 0.f;
        owt[i] = lab[i] >= 0 ? ow : 0.f;
        if (fg) {                                                     // utils/boxes.py:199-230, weights (1, 1, 1, 1), float32
            const float4 ex = rpn_anchor(g, l, idx);
            const float4 q = __ldg(gt + g.gt_begin[n] + __ldg(am + idx));
            const float ew = __fadd_rn(__fsub_rn(ex.z, ex.x), 1.f), eh = __fadd_rn(__fsub_rn(ex.w, ex.y), 1.f);
            const float ecx = __fadd_rn(ex.x, __fmul_rn(0.5f, ew)), ecy = __fadd_rn(ex.y, __fmul_rn(0.5f, eh));
            const float gw = __fadd_rn(__fsub_rn(q.z, q.x), 1.f), gh = __fadd_rn(__fsub_rn(q.w, q.y), 1.f);
            const float gcx = __fadd_rn(q.x, __fmul_rn(0.5f, gw)), gcy = __fadd_rn(q.y, __fmul_rn(0.5f, gh));
            tg[0][i] = __fdiv_rn(__fsub_rn(gcx, ecx), ew);
            tg[1][i] = __fdiv_rn(__fsub_rn(gcy, ecy), eh);
            tg[2][i] = logf(__fdiv_rn(gw, ew));
            tg[3][i] = logf(__fdiv_rn(gh, eh));
        }
    }
    const long long lplane = ((long long)n * A + a) * F2 + p0;
    const long long tplane = ((long long)n * 4 * A + 4 * a) * F2 + p0;
    if (VEC) {
        *reinterpret_cast<int4*>(o.labels[l] + lplane) = make_int4(lab[0], lab[1], lab[2], lab[3]);
        const float4 wi = make_float4(iw[0], iw[1], iw[2], iw[3]), wo = make_float4(owt[0], owt[1], owt[2], owt[3]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const long long off = tplane + (long long)k * F2;
            *reinterpret_cast<float4*>(o.targets[l] + off) = make_float4(tg[k][0], tg[k][1], tg[k][2], tg[k][3]);
            *reinterpret_cast<float4*>(o.inside[l] + off) = wi;
            *reinterpret_cast<float4*>(o.outside[l] + off) = wo;
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (p0 + i >= F2) continue;
            o.labels[l][lplane + i] = lab[i];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const long long off = tplane + (long long)k * F2 + i;
                o.targets[l][off] = tg[k][i]; o.inside[l][off] = iw[i]; o.outside[l][off] = owt[i];
            }
        }
    }
}

__global__ void __launch_bounds__(256)
rpn_emit_kernel(const __grid_constant__ RpnGeom g, const __grid_constant__ RpnOut o, const float4* __restrict__ gt, long long tpad,
                const unsigned char* __restrict__ flags, const int* __restrict__ argmax, const int* __restrict__ num_examples) {
    const int n = blockIdx.y, u = blockIdx.x * 256 + threadIdx.x;
    if (u >= o.unit_start[g.num_levels]) return;
    int l = 0;
    while (l + 1 < g.num_levels && u >= o.unit_start[l + 1]) ++l;
    const int F2 = g.F[l] * g.F[l], Q = (F2 + 3) / 4, local = u - o.unit_start[l];
    const int a = local / Q, p0 = (local - a * Q) * 4;
    const int ne = __ldg(num_examples + n);
    const float ow = ne > 0 ? (float)__drcp_rn((double)ne) : 0.f;    // float32(1.0 / num_examples), rpn.py:212-214
    const unsigned char* fl = flags + n * tpad;
    const int* am = argmax + (long long)n * g.total;
    if (F2 % 4 == 0) rpn_emit_unit<true>(g, o, n, l, a, p0, gt, fl, am, ow);
    else rpn_emit_unit<false>(g, o, n, l, a, p0, gt, fl, am, ow);
}

struct RpnWs {
    unsigned* colmax; unsigned char* flags; int *argmax, *fg_list, *bg_list, *blk_counts, *num_examples;
    long long tpad; int nblk;
};

size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

// workspace carve-up: colmax (sum G) | flags (N * tpad bytes) | argmax, fg_list, bg_list (N * T each) | blk_counts | num_examples
size_t rpn_ws_layout(int N, int T, int sumG, RpnWs* w, void* base) {
    const long long tpad = ((long long)T + 15) & ~15LL;
    const int nblk = (T + kRpnTile - 1) / kRpnTile;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off += align256(bytes); return (char*)base + o; };
    RpnWs v;
    v.colmax = (unsigned*)take(sizeof(unsigned) * (size_t)(sumG > 0 ? sumG : 1));
    v.flags = (unsigned char*)take((size_t)N * tpad);
    v.argmax = (int*)take(sizeof(int) * (size_t)N * T);
    v.fg_list = (int*)take(sizeof(int) * (size_t)N * T);
    v.bg_list = (int*)take(sizeof(int) * (size_t)N * T);
    v.blk_counts = (int*)take(sizeof(int) * 3 * (size_t)N * nblk);
    v.num_examples = (int*)take(sizeof(int) * (size_t)N);
    v.tpad = tpad; v.nblk = nblk;
    if (w) *w = v;
    return off;
}

// level / image tables -> RpnGeom; false on any argument error
bool rpn_geom(int L, const int* F, const int* A, const double* strides, const double* cell, int N, const double* im_sizes,
              const int* gt_begin, double straddle, RpnGeom* g) {
    if (L < 1 || L > kRpnMaxLevels || N < 1 || N > kRpnMaxImages || !F || !A || !strides || !cell || !im_sizes || !gt_begin) return false;
    RpnGeom v{};
    v.num_levels = L; v.num_images = N;
    long long total = 0;
    int cells = 0;
    for (int l = 0; l < L; ++l) {
        if (F[l] < 1 || A[l] < 1 || F[l] > 46340) return false;
        if (cells + A[l] > kRpnMaxCellAnchors) return false;
        v.F[l] = F[l]; v.A[l] = A[l]; v.cell0[l] = cells; v.stride[l] = strides[l]; v.start[l] = (int)total;
        for (int a = 0; a < A[l]; ++a)
            for (int k = 0; k < 4; ++k) v.cell[cells + a][k] = cell[4 * (cells + a) + k];
        cells += A[l];
        total += (long long)F[l] * F[l] * A[l];
        if (total > (1LL << 30)) return false;
    }
    v.start[L] = (int)total; v.total = (int)total;
    v.keep_all = straddle < 0;
    v.xymin = (float)(-straddle);
    if (gt_begin[0] != 0) return false;
    for (int n = 0; n < N; ++n) {
        if (gt_begin[n + 1] <= gt_begin[n]) return false;                   // every image needs ground truth (rpn.py:144)
        v.xmax[n] = im_sizes[2 * n + 1] + straddle; v.ymax[n] = im_sizes[2 * n] + straddle;
        v.gt_begin[n] = gt_begin[n];
    }
    v.gt_begin[N] = gt_begin[N];
    *g = v;
    return true;
}

size_t rpn_workspace_bytes(int N, int T, int sumG) {
    if (N < 1 || N > kRpnMaxImages || T < 1 || sumG < 0) return 0;
    return rpn_ws_layout(N, T, sumG, nullptr, nullptr);
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_rpn_targets_workspace_bytes(int L, const int* F, const int* A, int N, int sumG) {
    if (L < 1 || L > kRpnMaxLevels || !F || !A) return 0;
    long long t = 0;
    for (int l = 0; l < L; ++l) {
        if (F[l] < 1 || A[l] < 1 || F[l] > 46340) return 0;
        t += (long long)F[l] * F[l] * A[l];
    }
    return t > (1LL << 30) ? 0 : rpn_workspace_bytes(N, (int)t, sumG);
}

int b200_rpn_labels(int L, const int* F, const int* A, const double* strides, const double* cell, int N, const double* im_sizes,
                    const int* gt_begin, const float* gt_boxes, double straddle, float pos_thresh, float neg_thresh, int* counts_out,
                    void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    RpnGeom g;
    if (!gt_boxes || !counts_out || !rpn_geom(L, F, A, strides, cell, N, im_sizes, gt_begin, straddle, &g)) return B200_ROI_EINVAL;
    const int sumG = gt_begin[N];
    if (!workspace || workspace_bytes < rpn_workspace_bytes(N, g.total, sumG)) return B200_ROI_EWORKSPACE;
    RpnWs w;
    rpn_ws_layout(N, g.total, sumG, &w, workspace);
    cudaMemsetAsync(w.colmax, 0, sizeof(unsigned) * (size_t)sumG, stream);
    const dim3 grid1((g.total + 255) / 256, N), grid2(w.nblk, N);
    rpn_colmax_kernel<<<grid1, 256, 0, stream>>>(g, (const float4*)gt_boxes, w.colmax);
    rpn_label_kernel<<<grid2, 256, 0, stream>>>(g, (const float4*)gt_boxes, w.colmax, pos_thresh, neg_thresh, w.tpad, w.flags, w.argmax,
                                                w.blk_counts);
    rpn_compact_kernel<<<grid2, 256, 0, stream>>>(g.total, w.tpad, w.flags, w.blk_counts, w.fg_list, w.bg_list, counts_out);
    return finish_launch(4);                                             // the memset counts as one
}

int b200_rpn_emit(int L, const int* F, const int* A, const double* strides, const double* cell, int N, const double* im_sizes,
                  const int* gt_begin, const float* gt_boxes, double straddle, const int* counts, const int* fg_disable, const int* dis_begin,
                  const int* bg_enable, const int* en_begin, void* workspace, size_t workspace_bytes, int* const* labels_out,
                  float* const* targets_out, float* const* inside_out, float* const* outside_out, b200_stream_t stream) {
    RpnGeom g;
    if (!gt_boxes || !counts || !dis_begin || !en_begin || !labels_out || !targets_out || !inside_out || !outside_out ||
        !rpn_geom(L, F, A, strides, cell, N, im_sizes, gt_begin, straddle, &g))
        return B200_ROI_EINVAL;
    RpnDraws d{};
    int max_draws = 0;
    if (dis_begin[0] != 0 || en_begin[0] != 0) return B200_ROI_EINVAL;
    for (int n = 0; n <= N; ++n) {
        d.dis_begin[n] = dis_begin[n]; d.en_begin[n] = en_begin[n];
        if (n < N) {
            if (dis_begin[n + 1] < dis_begin[n] || en_begin[n + 1] < en_begin[n]) return B200_ROI_EINVAL;
            max_draws = max(max_draws, dis_begin[n + 1] - dis_begin[n] + en_begin[n + 1] - en_begin[n]);
        }
    }
    if ((dis_begin[N] > 0 && !fg_disable) || (en_begin[N] > 0 && !bg_enable)) return B200_ROI_EINVAL;
    RpnOut o{};
    int units = 0;
    for (int l = 0; l < L; ++l) {
        if (!labels_out[l] || !targets_out[l] || !inside_out[l] || !outside_out[l]) return B200_ROI_EINVAL;
        o.labels[l] = labels_out[l]; o.targets[l] = targets_out[l]; o.inside[l] = inside_out[l]; o.outside[l] = outside_out[l];
        const bool vec = (F[l] * F[l]) % 4 == 0;
        if (vec && (((uintptr_t)labels_out[l] | (uintptr_t)targets_out[l] | (uintptr_t)inside_out[l] | (uintptr_t)outside_out[l]) & 15))
            return B200_ROI_EINVAL;                                           // the 16-byte stores need 16-byte aligned blobs
        o.unit_start[l] = units;
        units += A[l] * ((F[l] * F[l] + 3) / 4);
    }
    o.unit_start[L] = units;
    const int sumG = gt_begin[N];
    if (!workspace || workspace_bytes < rpn_workspace_bytes(N, g.total, sumG)) return B200_ROI_EWORKSPACE;
    RpnWs w;
    rpn_ws_layout(N, g.total, sumG, &w, workspace);
    rpn_scatter_draw_kernel<<<dim3((max(max_draws, 1) + 255) / 256, N), 256, 0, stream>>>(d, g.total, w.tpad, counts, fg_disable, bg_enable,
                                                                                           w.fg_list, w.bg_list, w.flags);
    rpn_count_kernel<<<N, 256, 0, stream>>>(d, g.total, w.tpad, counts, bg_enable, w.bg_list, w.flags, w.num_examples);
    rpn_emit_kernel<<<dim3((units + 255) / 256, N), 256, 0, stream>>>(g, o, (const float4*)gt_boxes, w.tpad, w.flags, w.argmax,
                                                                      w.num_examples);
    return finish_launch(3);
}

}  // extern "C"
