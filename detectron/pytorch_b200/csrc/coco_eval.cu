// coco_eval.cu -- COCO box, mask and keypoint evaluation on the device (the stages of pycocotools' COCOeval that the reference's
// json_dataset_evaluator calls: evaluate() and accumulate(); oracle/cocoeval.py restates them).
//
// The work is grouped per (image, category) pair; pairs are ordered image-major (sorted image ids, then category index), a
// pair's detections in results order, its ground truth in annotation order.
//   coco_rank_kernel        one CTA per pair: the stable descending-score rank of each detection (computeIoU / evaluateImg's
//                           mergesort), cut to maxDets[-1]: the pair's "entries" in rank order
//   coco_bbox_iou_kernel    one CTA per pair: maskApi bbIou in double
//   coco_oks_kernel         one CTA per pair: computeOks
//   coco_*_toggles_kernel   masks as bitmaps of the image's h * w pixels in column-major order: compressed strings
//                           (rleFrString), uncompressed counts and polygons (rleFrPoly, poly_walk.cuh) toggle the bit where a
//                           run starts;
//   coco_fill_kernel        one CTA per mask: a prefix XOR over the bitmap turns toggles into pixels, the union over an
//                           object's polygons (annToRLE's merge), its area and the span of non-zero words
//   coco_segm_iou_kernel    one warp per (entry, ground truth): popcount of the AND over the overlapping words (rleIou)
//   coco_match_kernel       one CTA per pair, one thread per (area range, threshold): evaluateImg's greedy matching
//   coco_accumulate_kernel  one CTA per (category, area range, maxDet): accumulate()'s tp / fp scans, precision envelope and
//                           the recall-threshold searches, over entries already ordered by a stable sort on the host side
// Every float64 step is an _rn intrinsic so no contraction changes a rounding.
#include <cfloat>

#include "poly_walk.cuh"

namespace b200 {

namespace {

constexpr int kCocoThreads = 256;
constexpr int kAccThreads = 512;
constexpr int kOksK = 17;
constexpr int kFlagCrowd = 1, kFlagIgnore = 2, kFlagIdNonzero = 4;

// ---- block scans ----------------------------------------------------------------------------------------------------------
template <typename T, typename Op>
__device__ __forceinline__ T block_inclusive_scan(T v, T* warp_sh, T& total, Op op, T identity) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v = op(y, v);
    }
    if (lane == 31) warp_sh[warp] = v;
    __syncthreads();
    if (warp == 0) {
        T w = lane < nw ? warp_sh[lane] : identity;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const T y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w = op(y, w);
        }
        if (lane < nw) warp_sh[lane] = w;
    }
    __syncthreads();
    if (warp > 0) v = op(warp_sh[warp - 1], v);
    total = warp_sh[nw - 1];
    __syncthreads();
    return v;
}

// ---- ranking ----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kCocoThreads)
coco_rank_kernel(const int* __restrict__ pair_det_begin, const int* __restrict__ pair_entry_begin, const double* __restrict__ det_score,
                 int* __restrict__ entry_det, int* __restrict__ entry_rank, double* __restrict__ entry_score) {
    const int p = blockIdx.x;
    const int d0 = pair_det_begin[p], d1 = pair_det_begin[p + 1];
    const int e0 = pair_entry_begin[p], ne = pair_entry_begin[p + 1] - e0;
    for (int d = d0 + threadIdx.x; d < d1; d += blockDim.x) {
        const double s = det_score[d];
        int r = 0;
        for (int j = d0; j < d1; ++j) {
            const double q = det_score[j];
            r += (q > s) || (q == s && j < d);
        }
        if (r < ne) { entry_det[e0 + r] = d; entry_rank[e0 + r] = r; entry_score[e0 + r] = s; }
    }
}

// ---- bbox ---------------------------------------------------------------------------------------------------------------
// maskApi bbIou: boxes (x, y, w, h) in double; u = the detection's box area for a crowd ground truth
__device__ __forceinline__ double bb_iou(double4 d, double4 g, bool crowd) {
    const double w = __dsub_rn(fmin(__dadd_rn(d.z, d.x), __dadd_rn(g.z, g.x)), fmax(d.x, g.x));
    if (w <= 0.0) return 0.0;
    const double h = __dsub_rn(fmin(__dadd_rn(d.w, d.y), __dadd_rn(g.w, g.y)), fmax(d.y, g.y));
    if (h <= 0.0) return 0.0;
    const double da = __dmul_rn(d.z, d.w), ga = __dmul_rn(g.z, g.w), i = __dmul_rn(w, h);
    const double u = crowd ? da : __dsub_rn(__dadd_rn(da, ga), i);
    return __ddiv_rn(i, u);
}

__global__ void __launch_bounds__(kCocoThreads)
coco_bbox_iou_kernel(const int* __restrict__ pair_gt_begin, const int* __restrict__ pair_entry_begin,
                     const long long* __restrict__ pair_iou_begin, const int* __restrict__ entry_det, const double4* __restrict__ det_box,
                     const double4* __restrict__ gt_box, const int* __restrict__ gt_flags, double* __restrict__ ious) {
    const int p = blockIdx.x;
    const int g0 = pair_gt_begin[p], G = pair_gt_begin[p + 1] - g0, e0 = pair_entry_begin[p], ne = pair_entry_begin[p + 1] - e0;
    double* out = ious + pair_iou_begin[p];
    for (int i = threadIdx.x; i < ne * G; i += blockDim.x) {
        const int r = i / G, g = i - r * G;
        out[i] = bb_iou(det_box[entry_det[e0 + r]], gt_box[g0 + g], gt_flags[g0 + g] & kFlagCrowd);
    }
}

// ---- keypoints ------------------------------------------------------------------------------------------------------------
struct OksVars {
    double v[kOksK];                                                     // (sigmas * 2) ** 2, computed by numpy on the host
};

// numpy's pairwise sum of n <= 17 float64 values: a plain loop below 8, else 8 accumulators and the rest in order
__device__ __forceinline__ double pairwise_sum(const double* a, int n) {
    if (n < 8) {
        double res = 0.0;
        for (int i = 0; i < n; ++i) res = __dadd_rn(res, a[i]);
        return res;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = a[j];
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], a[i + j]);
    }
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __dadd_rn(res, a[i]);
    return res;
}

__global__ void __launch_bounds__(kCocoThreads)
coco_oks_kernel(const __grid_constant__ OksVars vars, const int* __restrict__ pair_gt_begin, const int* __restrict__ pair_entry_begin,
                const long long* __restrict__ pair_iou_begin, const int* __restrict__ entry_det, const double* __restrict__ det_kp,
                const double* __restrict__ gt_kp, const double4* __restrict__ gt_box, const double* __restrict__ gt_area,
                double* __restrict__ ious) {
    const int p = blockIdx.x;
    const int g0 = pair_gt_begin[p], G = pair_gt_begin[p + 1] - g0, e0 = pair_entry_begin[p], ne = pair_entry_begin[p + 1] - e0;
    double* out = ious + pair_iou_begin[p];
    for (int i = threadIdx.x; i < ne * G; i += blockDim.x) {
        const int r = i / G, g = g0 + i - r * G;
        const double* d = det_kp + (long long)entry_det[e0 + r] * 3 * kOksK;
        const double* q = gt_kp + (long long)g * 3 * kOksK;
        int k1 = 0;
        for (int k = 0; k < kOksK; ++k) k1 += q[3 * k + 2] > 0.0;
        const double4 bb = gt_box[g];
        const double x0 = __dsub_rn(bb.x, bb.z), x1 = __dadd_rn(bb.x, __dmul_rn(bb.z, 2.0));
        const double y0 = __dsub_rn(bb.y, bb.w), y1 = __dadd_rn(bb.y, __dmul_rn(bb.w, 2.0));
        const double den = __dadd_rn(gt_area[g], DBL_EPSILON);           // area + np.spacing(1)
        double ex[kOksK];
        int n = 0;
        for (int k = 0; k < kOksK; ++k) {
            const double xd = d[3 * k], yd = d[3 * k + 1];
            double dx, dy;
            if (k1 > 0) {
                if (!(q[3 * k + 2] > 0.0)) continue;
                dx = __dsub_rn(xd, q[3 * k]); dy = __dsub_rn(yd, q[3 * k + 1]);
            } else {
                dx = __dadd_rn(fmax(0.0, __dsub_rn(x0, xd)), fmax(0.0, __dsub_rn(xd, x1)));
                dy = __dadd_rn(fmax(0.0, __dsub_rn(y0, yd)), fmax(0.0, __dsub_rn(yd, y1)));
            }
            const double e = __ddiv_rn(__ddiv_rn(__ddiv_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), vars.v[k]), den), 2.0);
            ex[n++] = exp(-e);
        }
        out[i] = __ddiv_rn(pairwise_sum(ex, n), (double)n);
    }
}

// ---- masks ------------------------------------------------------------------------------------------------------------------
struct SlotTable {
    const long long* word;                                               // first 32-bit word of each slot (n_slots + 1)
    const int2* hw;                                                      // (h, w) of each slot's image
};

__device__ __forceinline__ void toggle(unsigned* bits, long long pos) { atomicXor(bits + (pos >> 5), 1u << (pos & 31)); }

// rleFrString: one thread per string; each run boundary inside the image toggles its bit
__global__ void __launch_bounds__(kCocoThreads)
coco_string_toggles_kernel(int n, const int* __restrict__ slot, const long long* __restrict__ begin, const unsigned char* __restrict__ bytes,
                           SlotTable st, unsigned* __restrict__ words) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = slot[i];
    const int2 hw = st.hw[s];
    const long long total = (long long)hw.x * hw.y;
    unsigned* bits = words + st.word[s];
    long long pos = 0, end = begin[i + 1];
    unsigned c1 = 0, c2 = 0;                                             // cnts[m - 1], cnts[m - 2]
    int m = 0;
    for (long long p = begin[i]; p < end;) {
        long long x = 0;
        int k = 0;
        bool more = true;
        while (more && p < end) {
            const int c = (int)bytes[p] - 48;
            x |= (long long)(c & 0x1f) << (5 * k);
            more = c & 0x20;
            ++p; ++k;
            if (!more && (c & 0x10)) x |= -1LL << (5 * k);
        }
        if (m > 2) x += (long long)c2;
        const unsigned cnt = (unsigned)x;
        c2 = c1; c1 = cnt; ++m;
        pos += cnt;
        if (pos < total) toggle(bits, pos);
    }
}

// uncompressed counts (crowd ground truth): one thread per RLE
__global__ void __launch_bounds__(kCocoThreads)
coco_count_toggles_kernel(int n, const int* __restrict__ slot, const long long* __restrict__ begin, const unsigned* __restrict__ counts,
                          SlotTable st, unsigned* __restrict__ words) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int s = slot[i];
    const int2 hw = st.hw[s];
    const long long total = (long long)hw.x * hw.y;
    unsigned* bits = words + st.word[s];
    long long pos = 0;
    for (long long p = begin[i]; p < begin[i + 1]; ++p) {
        pos += counts[p];
        if (pos < total) toggle(bits, pos);
    }
}

// rleFrPoly in the image frame: one thread per polygon edge (vertex j -> j + 1 of its ring), plus the step from the previous
// edge's last walk point; a crossing at column xd, row yd toggles column-major position xd * h + yd
__global__ void __launch_bounds__(kCocoThreads)
coco_poly_toggles_kernel(int n_poly, const int* __restrict__ vtx_begin, const double* __restrict__ xy, const int* __restrict__ slot,
                         SlotTable st, unsigned* __restrict__ words) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= vtx_begin[n_poly]) return;
    int lo = 0, hi = n_poly - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (vtx_begin[mid] <= g) lo = mid; else hi = mid - 1;
    }
    const int v0 = vtx_begin[lo], k = vtx_begin[lo + 1] - v0, j = g - v0;
    const int s = slot[lo];
    const int2 hw = st.hw[s];
    const int h = hw.x, w = hw.y;
    const long long total = (long long)h * w;
    unsigned* bits = words + st.word[s];
    auto vertex = [&](int q) {                                           // (int)(5 * x + .5), C truncation
        const double* p = xy + 2LL * (v0 + q);
        return make_int2(__double2int_rz(__dadd_rn(__dmul_rn((double)poly::kUpsample, p[0]), 0.5)),
                         __double2int_rz(__dadd_rn(__dmul_rn((double)poly::kUpsample, p[1]), 0.5)));
    };
    auto emit = [&](int pu, int pv, int qu, int qv) {
        int xd, yd;
        if (!poly::crossing(pu, pv, qu, qv, h, w, xd, yd)) return;
        const long long pos = (long long)xd * h + yd;
        if (pos < total) toggle(bits, pos);
    };
    const int2 a = vertex(j), c = vertex((j + 1) % k);
    const poly::Edge e = poly::make_edge(a.x, a.y, c.x, c.y);
    poly::edge_crossings(e, w, emit);
    if (j > 0) {
        const int2 z = vertex(j - 1);
        const poly::Edge f = poly::make_edge(z.x, z.y, a.x, a.y);
        emit(poly::edge_u(f, f.n), poly::edge_v(f, f.n), poly::edge_u(e, 0), poly::edge_v(e, 0));
    }
}

// one CTA per mask: pixels = inclusive prefix XOR of the toggles (column-major, bit p & 31 of word p >> 5); a mask with several
// slots (an object's polygons) is their union, left in its first slot; area and the first / last non-zero word
__global__ void __launch_bounds__(kCocoThreads)
coco_fill_kernel(const int* __restrict__ mask_slot_begin, SlotTable st, unsigned* __restrict__ words, long long* __restrict__ mask_area,
                 int2* __restrict__ mask_range) {
    __shared__ unsigned s_par[kCocoThreads / 32];
    __shared__ unsigned long long s_area;
    __shared__ int s_lo, s_hi;
    const int mk = blockIdx.x, s0 = mask_slot_begin[mk], s1 = mask_slot_begin[mk + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int2 hw = st.hw[s0];
    const long long nbits = (long long)hw.x * hw.y, nw = (nbits + 31) >> 5;
    const unsigned tail = (nbits & 31) ? ((1u << (nbits & 31)) - 1u) : ~0u;
    unsigned* out = words + st.word[s0];
    if (threadIdx.x == 0) { s_area = 0ull; s_lo = INT_MAX; s_hi = -1; }
    unsigned long long area = 0ull;
    int wlo = INT_MAX, whi = -1;
    for (int s = s0; s < s1; ++s) {
        const unsigned* in = words + st.word[s];
        unsigned carry = 0;
        for (long long base = 0; base < nw; base += blockDim.x) {
            const long long i = base + threadIdx.x;
            const unsigned x = i < nw ? in[i] : 0u;
            const unsigned bal = __ballot_sync(0xffffffffu, __popc(x) & 1);
            if (lane == 0) s_par[warp] = __popc(bal) & 1;
            __syncthreads();
            unsigned before = carry ^ (__popc(bal & ((1u << lane) - 1u)) & 1);
            unsigned tile = 0;
            for (int q = 0; q < (int)(blockDim.x >> 5); ++q) {
                if (q < warp) before ^= s_par[q];
                tile ^= s_par[q];
            }
            __syncthreads();
            carry ^= tile;
            if (i < nw) {
                unsigned y = x;
                y ^= y << 1; y ^= y << 2; y ^= y << 4; y ^= y << 8; y ^= y << 16;
                if (before) y = ~y;
                if (i == nw - 1) y &= tail;
                if (s != s0) y |= out[i];
                out[i] = y;
                if (s == s1 - 1 && y) {
                    area += __popc(y);
                    wlo = min(wlo, (int)i); whi = max(whi, (int)i);
                }
            }
        }
    }
    if (area) atomicAdd(&s_area, area);
    if (whi >= 0) { atomicMin(&s_lo, wlo); atomicMax(&s_hi, whi); }
    __syncthreads();
    if (threadIdx.x == 0) {
        mask_area[mk] = (long long)s_area;
        mask_range[mk] = s_hi >= 0 ? make_int2(s_lo, s_hi) : make_int2(1, 0);
    }
}

// rleIou on the bitmaps: one warp per (entry, ground truth); i = popcount of the AND over the words both masks cover
// (the box pre-test of rleIou: masks whose spans do not meet score 0); u = the detection's area for a crowd ground truth
__global__ void __launch_bounds__(kCocoThreads)
coco_segm_iou_kernel(int p0, const int* __restrict__ pair_gt_begin, const int* __restrict__ pair_entry_begin,
                     const long long* __restrict__ pair_iou_begin, const int* __restrict__ entry_det, int det0, int gt0, int gt_mask0,
                     const int* __restrict__ mask_slot_begin, SlotTable st, const unsigned* __restrict__ words,
                     const long long* __restrict__ mask_area, const int2* __restrict__ mask_range, const int* __restrict__ gt_flags,
                     double* __restrict__ ious) {
    const int p = p0 + blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int g0 = pair_gt_begin[p], G = pair_gt_begin[p + 1] - g0, e0 = pair_entry_begin[p], ne = pair_entry_begin[p + 1] - e0;
    double* out = ious + pair_iou_begin[p];
    for (int i = warp; i < ne * G; i += nwarps) {
        const int r = i / G, g = g0 + i - r * G;
        const int dm = entry_det[e0 + r] - det0, gm = gt_mask0 + g - gt0;
        const int2 dr = mask_range[dm], gr = mask_range[gm];
        const int lo = max(dr.x, gr.x), hi = min(dr.y, gr.y);
        const unsigned* a = words + st.word[mask_slot_begin[dm]];
        const unsigned* b = words + st.word[mask_slot_begin[gm]];
        unsigned long long n = 0;
        for (int w = lo + lane; w <= hi; w += 32) n += __popc(a[w] & b[w]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
        if (lane == 0) {
            double v = 0.0;
            if (n) {
                const long long da = mask_area[dm], ga = mask_area[gm];
                const long long u = (gt_flags[g] & kFlagCrowd) ? da : da + ga - (long long)n;
                v = __ddiv_rn((double)n, (double)u);
            }
            out[i] = v;
        }
    }
}

// ---- matching -----------------------------------------------------------------------------------------------------------
struct MatchParams {
    int T, A;
    double thr[16];
    double area_lo[8], area_hi[8];
};

// evaluateImg for maxDets[-1], one thread per (area range a, threshold t).  Ground truth is visited stably with the
// non-ignored first; entry_flags[a][e] gets bit t when the entry matched a ground truth with a non-zero id (dtMatches != 0)
// and bit 16 + t when it is ignored; npig[cat][a] += the pair's non-ignored ground truth
__global__ void __launch_bounds__(64)
coco_match_kernel(const __grid_constant__ MatchParams mp, const int* __restrict__ pair_gt_begin, const int* __restrict__ pair_entry_begin,
                  const long long* __restrict__ pair_iou_begin, const int* __restrict__ pair_cat, const int* __restrict__ entry_det,
                  const double* __restrict__ det_area, const double* __restrict__ gt_area, const int* __restrict__ gt_flags,
                  const double* __restrict__ ious, int num_entries, unsigned* __restrict__ entry_flags, int* __restrict__ npig) {
    extern __shared__ unsigned char gtm[];                              // (A * T) x G matched flags
    const int p = blockIdx.x;
    const int g0 = pair_gt_begin[p], G = pair_gt_begin[p + 1] - g0, e0 = pair_entry_begin[p], ne = pair_entry_begin[p + 1] - e0;
    const int AT = mp.A * mp.T;
    for (int i = threadIdx.x; i < AT * G; i += blockDim.x) gtm[i] = 0;
    __syncthreads();
    if (threadIdx.x >= AT) return;
    const int a = threadIdx.x / mp.T, t = threadIdx.x - a * mp.T;
    const double lo = mp.area_lo[a], hi = mp.area_hi[a];
    auto ignored = [&](int g) {
        const double ar = gt_area[g0 + g];
        return (gt_flags[g0 + g] & kFlagIgnore) || ar < lo || ar > hi;
    };
    if (t == 0) {
        int n = 0;
        for (int g = 0; g < G; ++g) n += !ignored(g);
        if (n) atomicAdd(npig + pair_cat[p] * mp.A + a, n);
    }
    unsigned char* my = gtm + threadIdx.x * G;
    const double* iou = ious + pair_iou_begin[p];
    const double t0 = fmin(mp.thr[t], 1.0 - 1e-10);
    for (int r = 0; r < ne; ++r) {
        const double* row = iou + (long long)r * G;
        double best = t0;
        int m = -1;
        bool m_ign = false;
        for (int pass = 0; pass < 2; ++pass) {
            for (int g = 0; g < G; ++g) {
                const bool ig = ignored(g);
                if (ig != (pass == 1)) continue;
                if (my[g] && !(gt_flags[g0 + g] & kFlagCrowd)) continue;
                if (m > -1 && !m_ign && ig) { pass = 2; break; }
                const double v = row[g];
                if (v < best) continue;
                best = v; m = g; m_ign = ig;
            }
        }
        const int e = e0 + r;
        bool matched_id = false, dt_ig = false;
        if (m >= 0) {
            my[m] = 1;
            matched_id = gt_flags[g0 + m] & kFlagIdNonzero;
            dt_ig = m_ign;
        }
        if (!matched_id) {
            const double da = det_area[entry_det[e]];
            if (da < lo || da > hi) dt_ig = true;
        }
        const unsigned bits = ((unsigned)matched_id << t) | ((unsigned)dt_ig << (16 + t));
        if (bits) atomicOr(entry_flags + (long long)a * num_entries + e, bits);
    }
}

// ---- accumulation ---------------------------------------------------------------------------------------------------------
struct AccParams {
    int K, A, M, T, R;
    int max_dets[8];
};

constexpr int kAccBits = 21;                                             // keep | tp | fp packed in one 64-bit scan value
constexpr unsigned long long kAccMask = (1ull << kAccBits) - 1ull;

// accumulate() for one (category k, area range a, maxDet m): the category's entries, already in stable descending-score order
// (image order, then rank, among ties), kept when rank < maxDet; per threshold the cumulative tp / fp (exact integers, so the
// float64 cumsum of the reference is the same), rc = tp / npig, pr = tp / (fp + tp + eps), the suffix maximum of pr and
// searchsorted(rc, recThrs, 'left')
__global__ void __launch_bounds__(kAccThreads)
coco_accumulate_kernel(const __grid_constant__ AccParams ap, const int* __restrict__ cat_entry_begin, const int* __restrict__ cat_pairs,
                       const int* __restrict__ order, const int* __restrict__ entry_rank, const double* __restrict__ entry_score,
                       const unsigned* __restrict__ entry_flags, int num_entries, const int* __restrict__ npig,
                       const double* __restrict__ rec_thrs, int* __restrict__ s_tp, double* __restrict__ s_pr, double* __restrict__ s_sc,
                       double* __restrict__ precision, double* __restrict__ recall, double* __restrict__ scores) {
    __shared__ unsigned long long sh_u[kAccThreads / 32];
    __shared__ double sh_d[kAccThreads / 32];
    const int k = blockIdx.x, a = blockIdx.y, m = blockIdx.z;
    if (cat_pairs[k] == 0) return;                                       // no image has ground truth or detections: -1
    const int np = npig[k * ap.A + a];
    if (np == 0) return;
    const int max_det = ap.max_dets[m];
    const int c0 = cat_entry_begin[k], n = cat_entry_begin[k + 1] - c0;
    const long long sbase = ((long long)a * ap.M + m) * num_entries + c0;
    int* tp_buf = s_tp + sbase;
    double* pr_buf = s_pr + sbase;
    double* sc_buf = s_sc + sbase;
    const unsigned* flags = entry_flags + (long long)a * num_entries;
    const double npd = (double)np;
    for (int t = 0; t < ap.T; ++t) {
        unsigned long long carry = 0;
        for (int base = 0; base < n; base += blockDim.x) {
            const int i = base + threadIdx.x;
            unsigned long long v = 0;
            int e = -1;
            if (i < n) {
                e = order[c0 + i];
                if (entry_rank[e] < max_det) {
                    const unsigned f = flags[e];
                    const bool mt = (f >> t) & 1u, ig = (f >> (16 + t)) & 1u;
                    v = (1ull << (2 * kAccBits)) | ((unsigned long long)(mt && !ig) << kAccBits) | (unsigned long long)(!mt && !ig);
                } else {
                    e = -1;
                }
            }
            unsigned long long tot;
            const unsigned long long incl = carry + block_inclusive_scan(v, sh_u, tot, [](unsigned long long x, unsigned long long y) { return x + y; }, 0ull);
            if (e >= 0) {
                const int j = (int)(incl >> (2 * kAccBits)) - 1;
                const int tp = (int)((incl >> kAccBits) & kAccMask), fp = (int)(incl & kAccMask);
                tp_buf[j] = tp;
                pr_buf[j] = __ddiv_rn((double)tp, __dadd_rn(__dadd_rn((double)fp, (double)tp), DBL_EPSILON));
                sc_buf[j] = entry_score[e];
            }
            carry += tot;
        }
        const int nd = (int)(carry >> (2 * kAccBits));
        __syncthreads();
        // suffix maximum of pr, tiles from the end; thread 0 holds the highest position of its tile
        double run = -INFINITY;
        for (int hi = nd; hi > 0; hi -= blockDim.x) {
            const int i = hi - 1 - (int)threadIdx.x;
            double x = i >= 0 ? pr_buf[i] : -INFINITY;
            double tot;
            x = fmax(run, block_inclusive_scan(x, sh_d, tot, [](double u, double w) { return fmax(u, w); }, -(double)INFINITY));
            if (i >= 0) pr_buf[i] = x;
            run = fmax(run, tot);
        }
        __syncthreads();
        const long long rbase = (((long long)t * ap.K + k) * ap.A + a) * ap.M + m;
        if (threadIdx.x == 0) recall[rbase] = nd ? __ddiv_rn((double)tp_buf[nd - 1], npd) : 0.0;
        for (int r = threadIdx.x; r < ap.R; r += blockDim.x) {
            const double thr = rec_thrs[r];
            int lo = 0, hi = nd;                                         // first j with tp_j / npig >= thr
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (__ddiv_rn((double)tp_buf[mid], npd) >= thr) hi = mid; else lo = mid + 1;
            }
            const long long o = ((((long long)t * ap.R + r) * ap.K + k) * ap.A + a) * ap.M + m;
            precision[o] = lo < nd ? pr_buf[lo] : 0.0;
            scores[o] = lo < nd ? sc_buf[lo] : 0.0;
        }
        __syncthreads();
    }
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_coco_rank(int num_pairs, const int* pair_det_begin, const int* pair_entry_begin, const double* det_score, int* entry_det, int* entry_rank,
                   double* entry_score, b200_stream_t stream) {
    if (num_pairs < 0 || (num_pairs > 0 && (!pair_det_begin || !pair_entry_begin || !det_score || !entry_det || !entry_rank || !entry_score)))
        return B200_ROI_EINVAL;
    if (num_pairs == 0) return B200_ROI_OK;
    coco_rank_kernel<<<num_pairs, kCocoThreads, 0, stream>>>(pair_det_begin, pair_entry_begin, det_score, entry_det, entry_rank, entry_score);
    return finish_launch();
}

int b200_coco_bbox_iou(int num_pairs, const int* pair_gt_begin, const int* pair_entry_begin, const long long* pair_iou_begin, const int* entry_det,
                       const double* det_box, const double* gt_box, const int* gt_flags, double* ious, b200_stream_t stream) {
    if (num_pairs < 0 || (num_pairs > 0 && (!pair_gt_begin || !pair_entry_begin || !pair_iou_begin || !entry_det || !det_box || !gt_box ||
                                            !gt_flags || !ious)))
        return B200_ROI_EINVAL;
    if (((uintptr_t)det_box | (uintptr_t)gt_box) & 15) return B200_ROI_EINVAL;
    if (num_pairs == 0) return B200_ROI_OK;
    coco_bbox_iou_kernel<<<num_pairs, kCocoThreads, 0, stream>>>(pair_gt_begin, pair_entry_begin, pair_iou_begin, entry_det,
                                                                 (const double4*)det_box, (const double4*)gt_box, gt_flags, ious);
    return finish_launch();
}

int b200_coco_oks(int num_pairs, const double* vars_host, const int* pair_gt_begin, const int* pair_entry_begin, const long long* pair_iou_begin,
                  const int* entry_det, const double* det_kp, const double* gt_kp, const double* gt_box, const double* gt_area, double* ious,
                  b200_stream_t stream) {
    if (num_pairs < 0 || !vars_host || (num_pairs > 0 && (!pair_gt_begin || !pair_entry_begin || !pair_iou_begin || !entry_det || !det_kp ||
                                                          !gt_kp || !gt_box || !gt_area || !ious)))
        return B200_ROI_EINVAL;
    if ((uintptr_t)gt_box & 15) return B200_ROI_EINVAL;
    if (num_pairs == 0) return B200_ROI_OK;
    OksVars v;
    for (int k = 0; k < kOksK; ++k) v.v[k] = vars_host[k];
    coco_oks_kernel<<<num_pairs, kCocoThreads, 0, stream>>>(v, pair_gt_begin, pair_entry_begin, pair_iou_begin, entry_det, det_kp, gt_kp,
                                                            (const double4*)gt_box, gt_area, ious);
    return finish_launch();
}

int b200_coco_masks(unsigned* words, long long num_words, int num_slots, const long long* slot_word, const int* slot_hw, int n_str,
                    const int* str_slot, const long long* str_begin, const unsigned char* str_bytes, int n_cnt, const int* cnt_slot,
                    const long long* cnt_begin, const unsigned* counts, int n_poly, int num_vertices, const int* poly_slot, const int* vtx_begin,
                    const double* xy, int n_masks, const int* mask_slot_begin, long long* mask_area, int* mask_range, b200_stream_t stream) {
    if (num_slots < 0 || n_str < 0 || n_cnt < 0 || n_poly < 0 || n_masks < 0 || num_words < 0 || num_vertices < 0) return B200_ROI_EINVAL;
    if (n_masks == 0) return B200_ROI_OK;
    if (!words || !slot_word || !slot_hw || !mask_slot_begin || !mask_area || !mask_range || (n_str && (!str_slot || !str_begin || !str_bytes)) ||
        (n_cnt && (!cnt_slot || !cnt_begin || !counts)) || (n_poly && (!poly_slot || !vtx_begin || !xy)))
        return B200_ROI_EINVAL;
    if (((uintptr_t)slot_hw | (uintptr_t)mask_range) & 7) return B200_ROI_EINVAL;
    const SlotTable st{slot_word, (const int2*)slot_hw};
    int launches = 0;
    if (cudaMemsetAsync(words, 0, (size_t)num_words * sizeof(unsigned), stream) != cudaSuccess) return finish_launch(0);
    if (n_str) { coco_string_toggles_kernel<<<(n_str + kCocoThreads - 1) / kCocoThreads, kCocoThreads, 0, stream>>>(n_str, str_slot, str_begin, str_bytes, st, words); ++launches; }
    if (n_cnt) { coco_count_toggles_kernel<<<(n_cnt + kCocoThreads - 1) / kCocoThreads, kCocoThreads, 0, stream>>>(n_cnt, cnt_slot, cnt_begin, counts, st, words); ++launches; }
    if (n_poly && num_vertices) {
        coco_poly_toggles_kernel<<<(num_vertices + kCocoThreads - 1) / kCocoThreads, kCocoThreads, 0, stream>>>(n_poly, vtx_begin, xy, poly_slot, st, words);
        ++launches;
    }
    coco_fill_kernel<<<n_masks, kCocoThreads, 0, stream>>>(mask_slot_begin, st, words, mask_area, (int2*)mask_range);
    return finish_launch(launches + 1);
}

int b200_coco_segm_iou(int pair_begin, int num_pairs, const int* pair_gt_begin, const int* pair_entry_begin, const long long* pair_iou_begin,
                       const int* entry_det, int det0, int gt0, int gt_mask0, const int* mask_slot_begin, const long long* slot_word,
                       const int* slot_hw, const unsigned* words, const long long* mask_area, const int* mask_range, const int* gt_flags,
                       double* ious, b200_stream_t stream) {
    if (pair_begin < 0 || num_pairs < 0) return B200_ROI_EINVAL;
    if (num_pairs == 0) return B200_ROI_OK;
    if (!pair_gt_begin || !pair_entry_begin || !pair_iou_begin || !entry_det || !mask_slot_begin || !slot_word || !slot_hw || !words ||
        !mask_area || !mask_range || !gt_flags || !ious || (((uintptr_t)slot_hw | (uintptr_t)mask_range) & 7))
        return B200_ROI_EINVAL;
    const SlotTable st{slot_word, (const int2*)slot_hw};
    coco_segm_iou_kernel<<<num_pairs, kCocoThreads, 0, stream>>>(pair_begin, pair_gt_begin, pair_entry_begin, pair_iou_begin, entry_det, det0,
                                                                 gt0, gt_mask0, mask_slot_begin, st, words, mask_area,
                                                                 (const int2*)mask_range, gt_flags, ious);
    return finish_launch();
}

int b200_coco_match(int num_pairs, int T, const double* iou_thrs_host, int A, const double* area_rng_host, int max_gt, const int* pair_gt_begin,
                    const int* pair_entry_begin, const long long* pair_iou_begin, const int* pair_cat, const int* entry_det, const double* det_area,
                    const double* gt_area, const int* gt_flags, const double* ious, int num_entries, unsigned* entry_flags, int* npig,
                    b200_stream_t stream) {
    if (num_pairs < 0 || T < 1 || T > 16 || A < 1 || A > 8 || A * T > 64 || max_gt < 0 || num_entries < 0 || !iou_thrs_host || !area_rng_host)
        return B200_ROI_EINVAL;
    const size_t smem = (size_t)A * T * max_gt;
    if (smem > 200 * 1024) return B200_ROI_EINVAL;
    if (num_pairs == 0) return B200_ROI_OK;
    if (!pair_gt_begin || !pair_entry_begin || !pair_iou_begin || !pair_cat || !entry_det || !det_area || !gt_area || !gt_flags || !ious ||
        !entry_flags || !npig)
        return B200_ROI_EINVAL;
    MatchParams mp{};
    mp.T = T; mp.A = A;
    for (int t = 0; t < T; ++t) mp.thr[t] = iou_thrs_host[t];
    for (int a = 0; a < A; ++a) { mp.area_lo[a] = area_rng_host[2 * a]; mp.area_hi[a] = area_rng_host[2 * a + 1]; }
    if (const int rc = smem_opt_in(coco_match_kernel, smem)) return rc;
    coco_match_kernel<<<num_pairs, 64, smem, stream>>>(mp, pair_gt_begin, pair_entry_begin, pair_iou_begin, pair_cat, entry_det, det_area,
                                                       gt_area, gt_flags, ious, num_entries, entry_flags, npig);
    return finish_launch();
}

int b200_coco_accumulate(int K, int A, int M, int T, int R, const int* max_dets_host, const int* cat_entry_begin, const int* cat_pairs,
                         const int* order, const int* entry_rank, const double* entry_score, const unsigned* entry_flags, int num_entries,
                         int max_cat_entries, const int* npig, const double* rec_thrs, void* workspace, size_t workspace_bytes, double* precision, double* recall,
                         double* scores, b200_stream_t stream) {
    if (K < 1 || A < 1 || A > 8 || M < 1 || M > 8 || T < 1 || T > 16 || R < 1 || num_entries < 0 || max_cat_entries < 0 ||
        max_cat_entries > num_entries || max_cat_entries >= (1 << kAccBits) || !max_dets_host)
        return B200_ROI_EINVAL;
    if (!cat_entry_begin || !cat_pairs || !npig || !rec_thrs || !precision || !recall || !scores ||
        (num_entries > 0 && (!order || !entry_rank || !entry_score || !entry_flags)))
        return B200_ROI_EINVAL;
    const size_t need = (size_t)A * M * num_entries * (sizeof(int) + 2 * sizeof(double));
    if (need && (!workspace || workspace_bytes < need || ((uintptr_t)workspace & 7))) return B200_ROI_EWORKSPACE;
    AccParams ap{};
    ap.K = K; ap.A = A; ap.M = M; ap.T = T; ap.R = R;
    for (int m = 0; m < M; ++m) ap.max_dets[m] = max_dets_host[m];
    const size_t n = (size_t)A * M * num_entries;
    double* pr = (double*)workspace;
    double* sc = pr + n;
    int* tp = (int*)(sc + n);
    coco_accumulate_kernel<<<dim3(K, A, M), kAccThreads, 0, stream>>>(ap, cat_entry_begin, cat_pairs, order, entry_rank, entry_score, entry_flags,
                                                                      num_entries, npig, rec_thrs, tp, pr, sc, precision, recall, scores);
    return finish_launch();
}

}  // extern "C"
