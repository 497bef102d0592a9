// losses.cu -- RPN and Fast R-CNN training losses (lib/modeling/rpn_heads.py:130-161, lib/modeling/FPN.py:422-466,
// lib/modeling/fast_rcnn_heads.py:50-68 with lib/utils/net.py:15-32), forward and backward, one launch each.
//
// Every element term is evaluated with the float32 operations of the reference expression, in its order, through _rn
// intrinsics so that nvcc never contracts them into FMAs; no element is skipped for a zero weight, so a non-finite
// prediction under a zero weight gives NaN exactly where the reference's `0 * inf` / `0 * NaN` does.  The terms are summed
// in float64: per thread, then per CTA in a fixed tree, then the last CTA to finish (an integer ticket, no floating-point
// atomics) adds the per-CTA partials in CTA order.  The grid size depends only on the shapes, so the result is the same bit
// for bit from run to run.
#include <algorithm>
#include <climits>

#include "common.cuh"

namespace b200 {
namespace {

constexpr int kMaxLevels = B200_RPN_LOSS_MAX_LEVELS;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kPerThread = 8;                       // items per thread per chunk, loaded before any is evaluated
constexpr int kChunk = kThreads * kPerThread;
constexpr int kMaxCtas = 2 * kNumSMs;
constexpr size_t kTicketBytes = 256;                // the ticket word, padded so the partials start aligned
constexpr float kRpnBeta = (float)(1.0 / 9.0);      // beta = 1/9 (rpn_heads.py:159), as torch rounds the Python scalar

// ---- element terms -------------------------------------------------------------------------------------------------------

// net_utils.smooth_l1_loss for one element: d = p - t; i = w_in * d; s = |i| < beta;
// ((s * 0.5) * (i * i)) / beta + (1 - s) * (|i| - 0.5 * beta), times w_out.
__device__ __forceinline__ float smooth_l1(float p, float t, float wi, float wo, float beta) {
    float i = __fmul_rn(wi, __fsub_rn(p, t));
    float a = fabsf(i);
    float s = (a < beta) ? 1.f : 0.f;
    float quad = __fdiv_rn(__fmul_rn(__fmul_rn(s, 0.5f), __fmul_rn(i, i)), beta);
    float lin = __fmul_rn(__fsub_rn(1.f, s), __fsub_rn(a, __fmul_rn(0.5f, beta)));
    return __fmul_rn(wo, __fadd_rn(quad, lin));
}

// Its gradient w.r.t. p for an upstream gradient gn (already divided by N), through the reference's autograd graph:
// pow's 2 * i branch and abs's sgn branch (sgn(NaN) = 0), so a zero weight still gives NaN where i is not finite.
__device__ __forceinline__ float smooth_l1_grad(float p, float t, float wi, float wo, float beta, float gn) {
    float i = __fmul_rn(wi, __fsub_rn(p, t));
    float a = fabsf(i);
    float s = (a < beta) ? 1.f : 0.f;
    float dterm = __fmul_rn(gn, wo);
    float d_pow = __fmul_rn(__fmul_rn(__fdiv_rn(dterm, beta), __fmul_rn(s, 0.5f)), __fmul_rn(2.f, i));
    float sgn = (float)((0.f < i) - (i < 0.f));
    float d_abs = __fmul_rn(__fmul_rn(dterm, __fsub_rn(1.f, s)), sgn);
    return __fmul_rn(__fadd_rn(d_pow, d_abs), wi);
}

// binary_cross_entropy_with_logits' element before the weight: (1 - y) * x - log_sigmoid(x), log_sigmoid as torch's
// min(0, x) - log1p(exp(-|x|)).
__device__ __forceinline__ float bce_logits(float x, float y) {
    float mn = (x < 0.f) ? x : 0.f;
    float ls = __fsub_rn(mn, log1pf(expf(-fabsf(x))));
    return __fsub_rn(__fmul_rn(__fsub_rn(1.f, y), x), ls);
}

__device__ __forceinline__ float sigmoid(float x) { return __fdiv_rn(1.f, __fadd_rn(1.f, expf(-x))); }

// log_softmax of the pair (l0, l1) at class c: (x_c - max) - log(exp(l0 - max) + exp(l1 - max)).
__device__ __forceinline__ void log_softmax2(float l0, float l1, float& o0, float& o1) {
    float m = l0 > l1 ? l0 : l1;
    float lse = logf(__fadd_rn(expf(__fsub_rn(l0, m)), expf(__fsub_rn(l1, m))));
    o0 = __fsub_rn(__fsub_rn(l0, m), lse);
    o1 = __fsub_rn(__fsub_rn(l1, m), lse);
}

// ---- deterministic reduction ---------------------------------------------------------------------------------------------

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// Sum over the CTA in a fixed order; the result is valid in thread 0.  Every thread must call it.
__device__ double block_sum(double v, double* smem /* kWarps */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();                                 // smem may still be read by a previous call
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int k = 0; k < kWarps; ++k) s += smem[k];
    return s;
}

// After every CTA has written its `nvals` partials at partials[blockIdx.x * nvals + k]: true in the one CTA that finished last,
// which then sees them all.  The ticket wraps back to 0 in that CTA, so the workspace is ready for the next call.
__device__ bool last_cta(unsigned* ticket) {
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = atomicInc(ticket, gridDim.x - 1) == gridDim.x - 1;
    __syncthreads();
    if (is_last) __threadfence();
    return is_last;
}

// In the last CTA: totals[k] = sum over CTAs b (in CTA order per lane, then a fixed warp tree) of partials[b * nvals + k].
__device__ void final_sums(const double* partials, int nvals, double* totals) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = warp; k < nvals; k += kWarps) {
        double s = 0.0;
        for (int b = lane; b < (int)gridDim.x; b += 32) s += __ldcg(partials + (size_t)b * nvals + k);
        s = warp_sum(s);
        if (lane == 0) totals[k] = s;
    }
    __syncthreads();
}

// ---- RPN -----------------------------------------------------------------------------------------------------------------

// Segment 2 l is level l's classification items (one per anchor, (n, a, y, x)); segment 2 l + 1 its box items (one per
// (n, 4 a + k, y, x)).  A chunk lies in one segment; chunk c of the step is in segment s when
// seg_chunk_begin[s] <= c < seg_chunk_begin[s + 1].
struct RpnLossParams {
    b200_rpn_loss_level lv[kMaxLevels];
    int seg_items[2 * kMaxLevels];
    int seg_chunk_begin[2 * kMaxLevels + 1];
    int num_levels;
    int softmax;
    float fixed_divisor;
};

__device__ __forceinline__ int find_segment(const RpnLossParams& P, int chunk) {
    int s = 0;
    while (chunk >= P.seg_chunk_begin[s + 1]) ++s;
    return s;
}

// Offsets of classification item e of level L: the logit (class 0 for softmax), the class-1 logit and the label.
struct ClsAt {
    long long x0, x1, lab;
};

__device__ __forceinline__ ClsAt cls_at(const b200_rpn_loss_level& L, unsigned e) {
    const unsigned hw = (unsigned)L.h * (unsigned)L.w;
    const unsigned plane = e / hw, r = e - plane * hw;
    const unsigned y = r / (unsigned)L.w, x = r - y * (unsigned)L.w;
    const unsigned n = plane / (unsigned)L.num_anchors, a = plane - n * (unsigned)L.num_anchors;
    ClsAt o;
    o.x0 = (long long)e;
    o.x1 = 0;
    if (L.cls_channels != L.num_anchors) {          // softmax: (N, 2A, h, w), the pair (a, A + a)
        const long long base = ((long long)n * 2 * L.num_anchors + a) * hw + r;
        o.x0 = base;
        o.x1 = base + (long long)L.num_anchors * hw;
    }
    o.lab = ((long long)plane * L.label_h + y) * L.label_w + x;
    return o;
}

// Offsets of box item e: into bbox_pred and into the three target blobs.
__device__ __forceinline__ long long box_wide_at(const b200_rpn_loss_level& L, unsigned e) {
    const unsigned hw = (unsigned)L.hb * (unsigned)L.wb;
    const unsigned plane = e / hw, r = e - plane * hw;
    const unsigned y = r / (unsigned)L.wb, x = r - y * (unsigned)L.wb;
    return ((long long)plane * L.target_h + y) * L.target_w + x;
}

__global__ void __launch_bounds__(kThreads) rpn_loss_forward_kernel(const __grid_constant__ RpnLossParams P, unsigned* ticket,
                                                                   double* partials, float* losses_out, float* divisor_out) {
    __shared__ double red[kWarps];
    __shared__ double seg_sum[2 * kMaxLevels], seg_cnt[2 * kMaxLevels];
    const int nseg = 2 * P.num_levels;
    if (threadIdx.x < 2 * kMaxLevels) seg_sum[threadIdx.x] = seg_cnt[threadIdx.x] = 0.0;
    const int total = P.seg_chunk_begin[nseg];
    int cur = -1;
    double acc = 0.0, cnt = 0.0;
    for (int c = blockIdx.x; c < total; c += gridDim.x) {
        const int s = find_segment(P, c);
        if (s != cur) {                              // CTA-uniform: chunks of one CTA visit the segments in order
            if (cur >= 0) {
                double t = block_sum(acc, red), k = block_sum(cnt, red);
                if (threadIdx.x == 0) { seg_sum[cur] = t; seg_cnt[cur] = k; }
            }
            cur = s;
            acc = cnt = 0.0;
        }
        const b200_rpn_loss_level& L = P.lv[s >> 1];
        const int items = P.seg_items[s];
        const unsigned e0 = (unsigned)(c - P.seg_chunk_begin[s]) * kChunk + threadIdx.x;
        if ((s & 1) == 0) {
            float x0[kPerThread], x1[kPerThread];
            int lab[kPerThread];
#pragma unroll
            for (int j = 0; j < kPerThread; ++j) {
                const unsigned e = e0 + j * kThreads;
                x0[j] = x1[j] = 0.f;
                lab[j] = -1;
                if (e < (unsigned)items) {
                    ClsAt o = cls_at(L, e);
                    x0[j] = L.cls_logits[o.x0];
                    if (P.softmax) x1[j] = L.cls_logits[o.x1];
                    lab[j] = L.labels_wide[o.lab];
                }
            }
#pragma unroll
            for (int j = 0; j < kPerThread; ++j) {
                if (e0 + j * kThreads >= (unsigned)items) continue;
                if (P.softmax) {
                    // F.cross_entropy(ignore_index=-1): an ignored pair adds nothing; a label other than 0 / 1 is never an index
                    if (lab[j] == -1) continue;
                    float o0, o1;
                    log_softmax2(x0[j], x1[j], o0, o1);
                    acc += (lab[j] == 0) ? -(double)o0 : (lab[j] == 1) ? -(double)o1 : (double)__int_as_float(0x7fffffff);
                    cnt += 1.0;
                } else {
                    const float w = lab[j] >= 0 ? 1.f : 0.f;
                    acc += (double)__fmul_rn(bce_logits(x0[j], (float)lab[j]), w);
                    cnt += (double)w;
                }
            }
        } else {
            float p[kPerThread], t[kPerThread], wi[kPerThread], wo[kPerThread];
#pragma unroll
            for (int j = 0; j < kPerThread; ++j) {
                const unsigned e = e0 + j * kThreads;
                p[j] = t[j] = wi[j] = wo[j] = 0.f;
                if (e < (unsigned)items) {
                    const long long q = box_wide_at(L, e);
                    p[j] = L.bbox_pred[e];
                    t[j] = L.bbox_targets_wide[q];
                    wi[j] = L.bbox_inside_wide[q];
                    wo[j] = L.bbox_outside_wide[q];
                }
            }
#pragma unroll
            for (int j = 0; j < kPerThread; ++j)
                if (e0 + j * kThreads < (unsigned)items) acc += (double)smooth_l1(p[j], t[j], wi[j], wo[j], kRpnBeta);
        }
    }
    if (cur >= 0) {
        double t = block_sum(acc, red), k = block_sum(cnt, red);
        if (threadIdx.x == 0) { seg_sum[cur] = t; seg_cnt[cur] = k; }
    }
    __syncthreads();
    double* mine = partials + (size_t)blockIdx.x * 2 * nseg;
    for (int k = threadIdx.x; k < nseg; k += kThreads) {
        mine[2 * k] = seg_sum[k];
        mine[2 * k + 1] = seg_cnt[k];
    }
    if (!last_cta(ticket)) return;
    __shared__ double totals[4 * kMaxLevels];
    final_sums(partials, 2 * nseg, totals);
    if (threadIdx.x < P.num_levels) {
        const int l = threadIdx.x;
        // cls: sum / (count of non-ignored labels), or / RPN_BATCH_SIZE_PER_IM * IMS_PER_BATCH for the FPN sigmoid loss
        const float div = P.fixed_divisor > 0.f ? P.fixed_divisor : (float)totals[4 * l + 1];
        losses_out[2 * l] = __fdiv_rn((float)totals[4 * l], div);
        losses_out[2 * l + 1] = __fdiv_rn((float)totals[4 * l + 2], (float)P.lv[l].num_images);
        divisor_out[l] = div;
    }
}

__global__ void __launch_bounds__(kThreads) rpn_loss_backward_kernel(const __grid_constant__ RpnLossParams P, const float* grad_losses,
                                                                    const float* divisor) {
    const int total = P.seg_chunk_begin[2 * P.num_levels];
    for (int c = blockIdx.x; c < total; c += gridDim.x) {
        const int s = find_segment(P, c);
        const int l = s >> 1;
        const b200_rpn_loss_level& L = P.lv[l];
        const int items = P.seg_items[s];
        const unsigned e0 = (unsigned)(c - P.seg_chunk_begin[s]) * kChunk + threadIdx.x;
        if ((s & 1) == 0) {
            const float gw = __fdiv_rn(grad_losses[2 * l], divisor[l]);
#pragma unroll 4
            for (int j = 0; j < kPerThread; ++j) {
                const unsigned e = e0 + j * kThreads;
                if (e >= (unsigned)items) break;
                ClsAt o = cls_at(L, e);
                const int lab = L.labels_wide[o.lab];
                if (P.softmax) {
                    // log_softmax backward of nll_loss's gradient (-gw at the label, 0 elsewhere and on ignored pairs)
                    float o0, o1;
                    log_softmax2(L.cls_logits[o.x0], L.cls_logits[o.x1], o0, o1);
                    const float g0 = lab == 0 ? -gw : 0.f, g1 = lab == 1 ? -gw : 0.f;
                    const float gs = lab == -1 ? 0.f : -gw;
                    float d0 = __fsub_rn(g0, __fmul_rn(expf(o0), gs)), d1 = __fsub_rn(g1, __fmul_rn(expf(o1), gs));
                    if (lab < -1 || lab > 1) d0 = d1 = __int_as_float(0x7fffffff);
                    L.cls_grad[o.x0] = d0;
                    L.cls_grad[o.x1] = d1;
                } else {
                    const float w = lab >= 0 ? 1.f : 0.f;
                    const float x = L.cls_logits[o.x0];
                    L.cls_grad[o.x0] = __fmul_rn(__fmul_rn(__fsub_rn(sigmoid(x), (float)lab), gw), w);
                }
            }
        } else {
            const float gn = __fdiv_rn(grad_losses[2 * l + 1], (float)L.num_images);
#pragma unroll 4
            for (int j = 0; j < kPerThread; ++j) {
                const unsigned e = e0 + j * kThreads;
                if (e >= (unsigned)items) break;
                const long long q = box_wide_at(L, e);
                L.bbox_grad[e] = smooth_l1_grad(L.bbox_pred[e], L.bbox_targets_wide[q], L.bbox_inside_wide[q], L.bbox_outside_wide[q],
                                                kRpnBeta, gn);
            }
        }
    }
}

int rpn_params(int num_levels, const b200_rpn_loss_level* levels, int activation, float fixed_divisor, bool backward, RpnLossParams& P) {
    if (num_levels < 1 || num_levels > kMaxLevels || levels == nullptr || (activation != 0 && activation != 1)) return B200_ROI_EINVAL;
    P = RpnLossParams{};
    P.num_levels = num_levels;
    P.softmax = activation;
    P.fixed_divisor = activation == 0 ? fixed_divisor : 0.f;
    P.seg_chunk_begin[0] = 0;
    long long chunks = 0;
    for (int l = 0; l < num_levels; ++l) {
        const b200_rpn_loss_level& L = levels[l];
        P.lv[l] = L;
        if (L.num_images < 1 || L.num_anchors < 1 || L.h < 0 || L.w < 0 || L.hb < 0 || L.wb < 0) return B200_ROI_EINVAL;
        if (L.cls_channels != (activation ? 2 : 1) * L.num_anchors) return B200_ROI_EINVAL;
        if (L.label_h < L.h || L.label_w < L.w || L.target_h < L.hb || L.target_w < L.wb) return B200_ROI_EINVAL;
        const long long nc = (long long)L.num_images * L.num_anchors * L.h * L.w;
        const long long nb = (long long)L.num_images * 4 * L.num_anchors * L.hb * L.wb;
        const long long wide_l = (long long)L.num_images * L.num_anchors * L.label_h * L.label_w;
        const long long wide_t = (long long)L.num_images * 4 * L.num_anchors * L.target_h * L.target_w;
        if (nc * (activation ? 2 : 1) >= (1LL << 31) || nb >= (1LL << 31) || wide_l >= (1LL << 40) || wide_t >= (1LL << 40)) return B200_ROI_EINVAL;
        if ((nc && (!L.cls_logits || !L.labels_wide)) ||
            (nb && (!L.bbox_pred || !L.bbox_targets_wide || !L.bbox_inside_wide || !L.bbox_outside_wide)))
            return B200_ROI_EINVAL;
        if (backward && ((nc && !L.cls_grad) || (nb && !L.bbox_grad))) return B200_ROI_EINVAL;
        P.seg_items[2 * l] = (int)nc;
        P.seg_items[2 * l + 1] = (int)nb;
        chunks += (nc + kChunk - 1) / kChunk;
        P.seg_chunk_begin[2 * l + 1] = (int)chunks;
        chunks += (nb + kChunk - 1) / kChunk;
        P.seg_chunk_begin[2 * l + 2] = (int)chunks;
    }
    if (chunks >= (1LL << 31)) return B200_ROI_EINVAL;
    return B200_ROI_OK;
}

// ---- Fast R-CNN ----------------------------------------------------------------------------------------------------------

struct RowCE {
    float m, lse;
};

// log_softmax statistics of row r (max, log of the sum of exp(x - max)), valid in every lane.
__device__ __forceinline__ RowCE row_logsumexp(const float* x, int C) {
    float m = -INFINITY;
    for (int c = threadIdx.x & 31; c < C; c += 32) m = fmaxf(m, x[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = threadIdx.x & 31; c < C; c += 32) s = __fadd_rn(s, expf(__fsub_rn(x[c], m)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __fadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    return RowCE{m, logf(s)};
}

__device__ __forceinline__ long long load_label(const void* labels, int label_is_int64, int r) {
    return label_is_int64 ? ((const long long*)labels)[r] : (long long)((const int*)labels)[r];
}

// torch's max(dim) index: the first maximal element, NaN counting as maximal.
__device__ __forceinline__ bool argmax_better(float a, int ia, float b, int ib) {
    const bool na = a != a, nb = b != b;
    if (na || nb) return na && (!nb || ia < ib);
    return a > b || (a == b && ia < ib);
}

struct FastRcnnArgs {
    const float* cls;
    const float* bbox;
    const void* labels;
    const float* targets;
    const float* inside;
    const float* outside;
    int R, C, B, label_is_int64;
};

__global__ void __launch_bounds__(kThreads) fast_rcnn_loss_forward_kernel(FastRcnnArgs a, unsigned* ticket, double* partials,
                                                                         float* losses_out, float* accuracy_out) {
    __shared__ double red[kWarps];
    const int lane = threadIdx.x & 31;
    double ce = 0.0, hits = 0.0, bb = 0.0;
    for (int r = blockIdx.x * kWarps + (threadIdx.x >> 5); r < a.R; r += gridDim.x * kWarps) {
        const float* x = a.cls + (size_t)r * a.C;
        const RowCE st = row_logsumexp(x, a.C);
        const long long t = load_label(a.labels, a.label_is_int64, r);
        const bool valid = t >= 0 && t < a.C;
        float best = 0.f;
        int bi = INT_MAX;                            // no element yet
        for (int c = lane; c < a.C; c += 32)
            if (bi == INT_MAX || argmax_better(x[c], c, best, bi)) { best = x[c]; bi = c; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi != INT_MAX && (bi == INT_MAX || argmax_better(ob, oi, best, bi))) { best = ob; bi = oi; }
        }
        if (lane == 0) {
            // -log_softmax(x)[t]; a label outside [0, C) is never an index: the loss is NaN
            ce += valid ? -(double)__fsub_rn(__fsub_rn(x[t], st.m), st.lse) : (double)__int_as_float(0x7fffffff);
            hits += (valid && bi == (int)t) ? 1.0 : 0.0;
        }
        const size_t o = (size_t)r * a.B;
        for (int c = lane; c < a.B; c += 32) bb += (double)smooth_l1(a.bbox[o + c], a.targets[o + c], a.inside[o + c], a.outside[o + c], 1.f);
    }
    const double s_ce = block_sum(ce, red), s_hits = block_sum(hits, red), s_bb = block_sum(bb, red);
    if (threadIdx.x == 0) {
        partials[3 * blockIdx.x] = s_ce;
        partials[3 * blockIdx.x + 1] = s_hits;
        partials[3 * blockIdx.x + 2] = s_bb;
    }
    if (!last_cta(ticket)) return;
    __shared__ double totals[3];
    final_sums(partials, 3, totals);
    if (threadIdx.x == 0) {
        const float R = (float)a.R;
        losses_out[0] = __fdiv_rn((float)totals[0], R);
        losses_out[1] = __fdiv_rn((float)totals[2], R);
        accuracy_out[0] = __fdiv_rn((float)totals[1], R);
    }
}

__global__ void __launch_bounds__(kThreads) fast_rcnn_loss_backward_kernel(FastRcnnArgs a, const float* grad_losses, float* cls_grad,
                                                                          float* bbox_grad) {
    const int lane = threadIdx.x & 31;
    const float R = (float)a.R;
    const float gw = cls_grad ? __fdiv_rn(grad_losses[0], R) : 0.f;
    const float gn = bbox_grad ? __fdiv_rn(grad_losses[1], R) : 0.f;
    for (int r = blockIdx.x * kWarps + (threadIdx.x >> 5); r < a.R; r += gridDim.x * kWarps) {
        if (cls_grad) {
            const float* x = a.cls + (size_t)r * a.C;
            const RowCE st = row_logsumexp(x, a.C);
            const long long t = load_label(a.labels, a.label_is_int64, r);
            const bool valid = t >= 0 && t < a.C;
            // log_softmax backward of nll_loss's gradient: (c == t ? -gw : 0) - exp(log_softmax(x)_c) * (-gw)
            for (int c = lane; c < a.C; c += 32) {
                const float lsm = __fsub_rn(__fsub_rn(x[c], st.m), st.lse);
                const float d = __fsub_rn(c == t ? -gw : 0.f, __fmul_rn(expf(lsm), -gw));
                cls_grad[(size_t)r * a.C + c] = valid ? d : __int_as_float(0x7fffffff);
            }
        }
        if (bbox_grad) {
            const size_t o = (size_t)r * a.B;
            for (int c = lane; c < a.B; c += 32)
                bbox_grad[o + c] = smooth_l1_grad(a.bbox[o + c], a.targets[o + c], a.inside[o + c], a.outside[o + c], 1.f, gn);
        }
    }
}

int fast_rcnn_args(int R, int C, int B, const float* cls, const float* bbox, const void* labels, int label_is_int64, const float* targets,
                   const float* inside, const float* outside, FastRcnnArgs& a) {
    if (R < 1 || C < 1 || B < 4 || B % 4 != 0 || (long long)R * C >= (1LL << 40) || (long long)R * B >= (1LL << 40)) return B200_ROI_EINVAL;
    if (!cls || !labels || (label_is_int64 != 0 && label_is_int64 != 1)) return B200_ROI_EINVAL;
    if (!bbox || !targets || !inside || !outside) return B200_ROI_EINVAL;
    a = FastRcnnArgs{cls, bbox, labels, targets, inside, outside, R, C, B, label_is_int64};
    return B200_ROI_OK;
}

int rows_grid(int R) { return (int)std::min<long long>(((long long)R + kWarps - 1) / kWarps, kMaxCtas); }

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_loss_workspace_bytes(int num_levels) {
    if (num_levels < 1 || num_levels > kMaxLevels) return 0;
    return kTicketBytes + (size_t)kMaxCtas * 4 * num_levels * sizeof(double);
}

int b200_rpn_loss_forward(int num_levels, const b200_rpn_loss_level* levels, int activation, float fixed_divisor, void* workspace,
                          size_t workspace_bytes, float* losses_out, float* divisor_out, b200_stream_t stream) {
    RpnLossParams P;
    int st = rpn_params(num_levels, levels, activation, fixed_divisor, false, P);
    if (st != B200_ROI_OK) return st;
    if (!losses_out || !divisor_out) return B200_ROI_EINVAL;
    if (!workspace || workspace_bytes < b200_loss_workspace_bytes(num_levels)) return B200_ROI_EWORKSPACE;
    const int chunks = P.seg_chunk_begin[2 * num_levels];
    const int grid = std::max(1, std::min(chunks, kMaxCtas));
    rpn_loss_forward_kernel<<<grid, kThreads, 0, stream>>>(P, (unsigned*)workspace, (double*)((char*)workspace + kTicketBytes), losses_out,
                                                          divisor_out);
    return finish_launch();
}

int b200_rpn_loss_backward(int num_levels, const b200_rpn_loss_level* levels, int activation, const float* grad_losses, const float* divisor,
                           b200_stream_t stream) {
    RpnLossParams P;
    int st = rpn_params(num_levels, levels, activation, 0.f, true, P);
    if (st != B200_ROI_OK) return st;
    if (!grad_losses || !divisor) return B200_ROI_EINVAL;
    const int chunks = P.seg_chunk_begin[2 * num_levels];
    if (chunks == 0) return B200_ROI_OK;
    rpn_loss_backward_kernel<<<std::min(chunks, 8 * kMaxCtas), kThreads, 0, stream>>>(P, grad_losses, divisor);
    return finish_launch();
}

int b200_fast_rcnn_loss_forward(int R, int C, int B, const float* cls, const float* bbox, const void* labels, int label_is_int64,
                                const float* targets, const float* inside, const float* outside, void* workspace, size_t workspace_bytes,
                                float* losses_out, float* accuracy_out, b200_stream_t stream) {
    FastRcnnArgs a;
    int st = fast_rcnn_args(R, C, B, cls, bbox, labels, label_is_int64, targets, inside, outside, a);
    if (st != B200_ROI_OK) return st;
    if (!losses_out || !accuracy_out) return B200_ROI_EINVAL;
    if (!workspace || workspace_bytes < b200_loss_workspace_bytes(1)) return B200_ROI_EWORKSPACE;
    fast_rcnn_loss_forward_kernel<<<rows_grid(R), kThreads, 0, stream>>>(a, (unsigned*)workspace, (double*)((char*)workspace + kTicketBytes),
                                                                        losses_out, accuracy_out);
    return finish_launch();
}

int b200_fast_rcnn_loss_backward(int R, int C, int B, const float* cls, const float* bbox, const void* labels, int label_is_int64,
                                 const float* targets, const float* inside, const float* outside, const float* grad_losses, float* cls_grad,
                                 float* bbox_grad, b200_stream_t stream) {
    FastRcnnArgs a;
    int st = fast_rcnn_args(R, C, B, cls, bbox, labels, label_is_int64, targets, inside, outside, a);
    if (st != B200_ROI_OK) return st;
    if (!grad_losses || (!cls_grad && !bbox_grad)) return B200_ROI_EINVAL;
    fast_rcnn_loss_backward_kernel<<<rows_grid(R), kThreads, 0, stream>>>(a, grad_losses, cls_grad, bbox_grad);
    return finish_launch();
}

}  // extern "C"
