// poly_walk.cuh -- pycocotools' rleFrPoly walk (oracle/masks.py restates it), shared by the Mask R-CNN training targets
// (mask_targets.cu, an M x M RoI frame) and the COCO evaluator's ground-truth masks (coco_eval.cu, the image frame).
//
// rleFrPoly upsamples every edge by 5 to integer points and emits a toggle wherever consecutive points cross a pixel column
// centre.  Along an edge the upsampled column u is monotone, so the single walk step that crosses column c (u from 5c + 2 to
// 5c + 3 or back) is found by bisection with the reference's own rounding: the work per edge is bounded by the columns it
// crosses, not by its upsampled length.
#pragma once
#include <climits>

#include "common.cuh"

namespace b200 {
namespace poly {

constexpr int kUpsample = 5;         // rleFrPoly's `scale`

// One edge of the upsampled walk, after rleFrPoly's swap.  Walk point d (0..n) is t = flip ? n - d : d.
struct Edge {
    int xs, ys, n;
    bool shallow, flip, degenerate;
    double s;
};

__device__ __forceinline__ Edge make_edge(int xs, int ys, int xe, int ye) {
    Edge e;
    const int dx = abs(xe - xs), dy = abs(ys - ye);
    e.shallow = dx >= dy;
    e.flip = (e.shallow && xs > xe) || (!e.shallow && ys > ye);
    if (e.flip) { int t = xs; xs = xe; xe = t; t = ys; ys = ye; ye = t; }
    e.xs = xs; e.ys = ys;
    e.n = e.shallow ? dx : dy;
    e.degenerate = dx == 0 && dy == 0;                                  // 0 / 0: the point's v is never a kept crossing's
    e.s = e.degenerate ? 0.0 : e.shallow ? __ddiv_rn((double)(ye - ys), (double)dx) : __ddiv_rn((double)(xe - xs), (double)dy);
    return e;
}

// (int)(a + s * t + .5): separate double roundings, C truncation
__device__ __forceinline__ int interp(int a, double s, int t) {
    return __double2int_rz(__dadd_rn(__dadd_rn((double)a, __dmul_rn(s, (double)t)), 0.5));
}

__device__ __forceinline__ int edge_u(const Edge& e, int d) {
    const int t = e.flip ? e.n - d : d;
    return e.shallow ? e.xs + t : interp(e.xs, e.s, t);
}

__device__ __forceinline__ int edge_v(const Edge& e, int d) {
    const int t = e.flip ? e.n - d : d;
    return e.shallow ? (e.degenerate ? INT_MIN : interp(e.ys, e.s, t)) : e.ys + t;   // INT_MIN: x86 cvttsd2si of NaN
}

// rleFrPoly's downsampling of the step (pu, pv) -> (qu, qv): true and column xd, row yd (0..h, h = the top of the next
// column) when the step is a kept crossing
__device__ __forceinline__ bool crossing(int pu, int pv, int qu, int qv, int h, int w, int& xd_out, int& yd_out) {
    if (qu == pu) return false;
    double xd = (double)(qu < pu ? qu : qu - 1);
    xd = __dsub_rn(__ddiv_rn(__dadd_rn(xd, 0.5), (double)kUpsample), 0.5);
    if (floor(xd) != xd || xd < 0.0 || xd > (double)(w - 1)) return false;
    double yd = (double)min(pv, qv);
    yd = __dsub_rn(__ddiv_rn(__dadd_rn(yd, 0.5), (double)kUpsample), 0.5);
    yd = yd < 0.0 ? 0.0 : yd > (double)h ? (double)h : yd;
    xd_out = (int)xd; yd_out = (int)ceil(yd);
    return true;
}

// floor(a / 5) for any sign
__device__ __forceinline__ int floordiv5(long long a) { return (int)(a >= 0 ? a / kUpsample : -((-a + kUpsample - 1) / kUpsample)); }

// every crossing inside one edge, passed to emit(pu, pv, qu, qv): the step that crosses column c is the first walk point
// past it, found by bisection; it is a crossing iff it lands exactly on 5c + 3 (rising) or 5c + 2 (falling)
template <typename Emit>
__device__ void edge_crossings(const Edge& e, int w, Emit emit) {
    if (e.n == 0) return;
    const int u0 = edge_u(e, 0), un = edge_u(e, e.n);
    if (u0 == un) return;
    const bool rising = un > u0;
    // rising: columns with 5c + 3 in (u0, un]; falling: 5c + 2 in [un, u0)
    const int clo = max(rising ? floordiv5((long long)u0 - 3) + 1 : floordiv5((long long)un - 2 + kUpsample - 1), 0);
    const int chi = min(rising ? floordiv5((long long)un - 3) : floordiv5((long long)u0 - 3), w - 1);
    for (int c = clo; c <= chi; ++c) {
        const int target = rising ? kUpsample * c + 3 : kUpsample * c + 2;
        int lo = 1, hi = e.n;                                             // point 0 is on the near side of the column
        while (lo < hi) {
            const int mid = lo + ((hi - lo) >> 1);
            const int u = edge_u(e, mid);
            if (rising ? u >= target : u <= target) hi = mid; else lo = mid + 1;
        }
        const int q = edge_u(e, lo);
        if (q != target) continue;                                        // the walk jumped over it: no crossing here
        emit(edge_u(e, lo - 1), edge_v(e, lo - 1), q, edge_v(e, lo));
    }
}

}  // namespace poly
}  // namespace b200
