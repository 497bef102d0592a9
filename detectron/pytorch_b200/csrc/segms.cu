// segms.cu -- test-time mask paste + COCO RLE (SURVEY.md 8f N3): the loop body of segm_results, lib/core/test.py:793-847
// (reference), for every detection of one image, without materialising the full-image masks.
//
// Per detection: the box is expanded by (M + 2) / M in float32 and truncated to int32 (lib/utils/boxes.py:233-249), the
// M x M soft mask is zero-padded to (M + 2)^2 and resized to the box with cv2.resize's float32 INTER_LINEAR arithmetic
// (IPP off), thresholded with a strict `>` and pasted into the image.  Only pixels inside the clipped box can be 1, so
// the run-length transitions are found by walking the window's columns; everything outside only lengthens runs.
//
// Resize arithmetic (cv2 imgproc resize.cpp, float32, every product and sum rounded on its own -- _rn intrinsics, no
// contraction):
//   per axis: scale = 1 / (dst / src) in double, f = float((d + .5) * scale - .5), s = floor(f), f -= s.  On the x axis a
//   position before the first / past the last source column is clamped to it with f = 0; on the y axis f is kept and the
//   two row indices s, s + 1 are clipped into the source.  Horizontal pass src[y][s] * (1 - f) + src[y][s + 1] * f, then
//   vertical pass row0 * (1 - g) + row1 * g.
//   Both axes shrinking by exactly 2 (30 -> 15 for M = 28) is cv2's INTER_AREA: its 4-lane vector loop covers the first
//   4 * floor(w / 4) columns of a row as ((a00 + a01) + (a10 + a11)) * .25, its scalar tail the rest as
//   (((a00 + a01) + a10) + a11) * .25.
//
// RLE (pycocotools rleEncode / rleToString): column-major counts starting with a run of zeros; the string encodes
// x = cnts[i] - (i > 2 ? cnts[i - 2] : 0) in 5-bit groups, low first, 0x20 = more, + 48.
//
// Two launches per image whatever the number of detections D: the sizes pass (one CTA per detection) counts transitions
// and string bytes and leaves each thread's scan state in the workspace; the emit pass re-walks each thread's chunk and
// writes counts and characters at their final places.
#include "common.cuh"
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

namespace b200 {

namespace {
constexpr int kSegmThreads = 256;
constexpr int kSegmMaxM = 64;
constexpr int kSegmMaxS = kSegmMaxM + 2;

struct SegmGeom {
    long long bx1, by1;        // origin of the int32 pasting box
    long long w, h;            // size the padded mask is resized to
    int x0, x1, y0, y1;        // paste window [y0, y1) x [x0, x1), empty when outside the image
    bool half;                 // both axes shrink by exactly 2: cv2's INTER_AREA
};

__device__ SegmGeom segm_geom(const float* __restrict__ box, int M, int im_h, int im_w) {
    const float scale = __double2float_rn(__ddiv_rn((double)(M + 2), (double)M));
    const float x1 = box[0], y1 = box[1], x2 = box[2], y2 = box[3];
    const float w_half = __fmul_rn(__fmul_rn(__fsub_rn(x2, x1), .5f), scale);
    const float h_half = __fmul_rn(__fmul_rn(__fsub_rn(y2, y1), .5f), scale);
    const float x_c = __fmul_rn(__fadd_rn(x2, x1), .5f), y_c = __fmul_rn(__fadd_rn(y2, y1), .5f);
    // __float2int_rz truncates like astype(np.int32) and saturates (NaN -> 0), so no box can index outside the mask
    const long long bx1 = __float2int_rz(__fsub_rn(x_c, w_half)), bx2 = __float2int_rz(__fadd_rn(x_c, w_half));
    const long long by1 = __float2int_rz(__fsub_rn(y_c, h_half)), by2 = __float2int_rz(__fadd_rn(y_c, h_half));
    SegmGeom g;
    g.bx1 = bx1; g.by1 = by1;
    g.w = bx2 - bx1 + 1 > 1 ? bx2 - bx1 + 1 : 1;
    g.h = by2 - by1 + 1 > 1 ? by2 - by1 + 1 : 1;
    const long long x0 = bx1 > 0 ? bx1 : 0, xe = bx2 + 1 < im_w ? bx2 + 1 : im_w;
    const long long y0 = by1 > 0 ? by1 : 0, ye = by2 + 1 < im_h ? by2 + 1 : im_h;
    const bool empty = x0 >= xe || y0 >= ye;
    g.x0 = empty ? 0 : (int)x0; g.x1 = empty ? 0 : (int)xe;
    g.y0 = empty ? 0 : (int)y0; g.y1 = empty ? 0 : (int)ye;
    g.half = 2 * g.w == M + 2 && 2 * g.h == M + 2;
    return g;
}

using Tap = Cv2Tap;

// one axis of cv2's INTER_LINEAR resized to a size (dsize): output index d of dst, source length src
__device__ __forceinline__ Tap linear_tap(long long d, long long dst, int src, bool clamp) {
    return cv2_linear_tap(d, __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src)), src, clamp);
}

// resized value at window pixel (dx, dy) of the box (tx: the x tap of column dx, unused on the 2x path)
__device__ __forceinline__ float segm_value(const float* pm, int S, const SegmGeom& g, const Tap& tx, long long dx, long long dy) {
    if (g.half) {
        const float* r0 = pm + 2 * dy * S + 2 * dx;
        const float* r1 = r0 + S;
        const float s = dx < (g.w & ~3LL) ? __fadd_rn(__fadd_rn(r0[0], r0[1]), __fadd_rn(r1[0], r1[1]))
                                          : __fadd_rn(__fadd_rn(__fadd_rn(r0[0], r0[1]), r1[0]), r1[1]);
        return __fmul_rn(s, .25f);
    }
    const Tap ty = linear_tap(dy, g.h, S, false);
    const float* q0 = pm + ty.s0 * S;
    const float* q1 = pm + ty.s1 * S;
    const float row0 = __fadd_rn(__fmul_rn(q0[tx.s0], tx.w0), __fmul_rn(q0[tx.s1], tx.w1));
    const float row1 = __fadd_rn(__fmul_rn(q1[tx.s0], tx.w0), __fmul_rn(q1[tx.s1], tx.w1));
    return __fadd_rn(__fmul_rn(row0, ty.w0), __fmul_rn(row1, ty.w1));
}

__device__ __forceinline__ bool segm_pixel(const float* pm, int S, const SegmGeom& g, int x, int y, float thresh) {
    const long long dx = x - g.bx1;
    const Tap tx = g.half ? Tap{} : linear_tap(dx, g.w, S, true);
    return segm_value(pm, S, g, tx, dx, y - g.by1) > thresh;
}

// zero-padded (M + 2)^2 mask of detection d in shared memory; a channel outside [0, Kc) reads as an all-zero mask
__device__ void load_padded(float* pm, const float* __restrict__ masks, const int* __restrict__ mask_class, int d, int Kc, int M) {
    const int S = M + 2;
    const int c = mask_class[d];
    const bool ok = c >= 0 && c < Kc;
    const float* src = masks + ((size_t)d * Kc + (ok ? c : 0)) * M * M;
    for (int i = threadIdx.x; i < S * S; i += blockDim.x) {
        const int r = i / S, q = i % S;
        pm[i] = (ok && r >= 1 && r <= M && q >= 1 && q <= M) ? src[(r - 1) * M + (q - 1)] : 0.f;
    }
}

// The window's column-major sequence: column x of the window contributes its (y1 - y0) pixels plus one trailing element
// at row y1 (value 0): linear position x * im_h + y1, which is (x + 1, 0) when y1 == im_h.  A transition is an element
// whose value differs from its predecessor in the image's column-major order.  The trailing element is skipped where the
// next column's first element is the same position (y0 == 0, y1 == im_h, x + 1 < x1) and at the end of the image.
template <typename OnTransition>
__device__ void segm_walk(const float* pm, int S, const SegmGeom& g, int im_h, int im_w, float thresh, long long e0, long long e1,
                          OnTransition on_transition) {
    if (e0 >= e1) return;
    const int Hn = g.y1 - g.y0, L = Hn + 1;
    long long xi = e0 / L;
    int yi = (int)(e0 % L);
    int x = g.x0 + (int)xi;
    Tap tx = g.half ? Tap{} : linear_tap(x - g.bx1, g.w, S, true);
    bool prev = yi > 0 ? segm_value(pm, S, g, tx, x - g.bx1, g.y0 + yi - 1 - g.by1) > thresh : false;
    const bool wraps = g.y0 == 0 && g.y1 == im_h;          // column x's first pixel follows column x - 1's last one
    for (long long e = e0; e < e1; ++e) {
        if (yi == 0) {
            if (e != e0) tx = g.half ? Tap{} : linear_tap(x - g.bx1, g.w, S, true);
            prev = (wraps && x > g.x0) ? segm_pixel(pm, S, g, x - 1, im_h - 1, thresh) : false;
        }
        bool cur = false, skip = false;
        if (yi < Hn) cur = segm_value(pm, S, g, tx, x - g.bx1, g.y0 + yi - g.by1) > thresh;
        else skip = g.y1 == im_h && ((g.y0 == 0 && x + 1 < g.x1) || x + 1 == im_w);
        if (cur != prev && !skip) on_transition(x * im_h + g.y0 + yi);
        prev = cur;
        if (++yi == L) { yi = 0; ++x; }
    }
}

// Transition positions T_1 < T_2 < ... after the virtual T_0 = 0; count i is T_{i+1} - T_i (the last one ends at im_h * im_w).
// A scan state holds the number of positions seen and the last three of them (p0 the latest).
struct Last3 {
    int n, p0, p1, p2;
};
struct Last3Op {
    __device__ Last3 operator()(const Last3& a, const Last3& b) const {
        Last3 r{a.n + b.n, b.p0, b.p1, b.p2};
        if (b.n == 2) r.p2 = a.p0;
        else if (b.n == 1) { r.p1 = a.p0; r.p2 = a.p1; }
        else if (b.n == 0) { r.p0 = a.p0; r.p1 = a.p1; r.p2 = a.p2; }
        return r;
    }
};
__device__ __forceinline__ void push(Last3& s, int q) { s.p2 = s.p1; s.p1 = s.p0; s.p0 = q; ++s.n; }

// the value rleToString encodes for the count that position q completes (or the final count, q = im_h * im_w)
__device__ __forceinline__ int rle_delta(const Last3& s, int q, int* count) {
    const int i = s.n - 1;
    *count = q - s.p0;
    return i > 2 ? *count - (s.p1 - s.p2) : *count;
}

__device__ __forceinline__ int rle_len(int x) {
    int n = 0;
    bool more = true;
    while (more) {
        const int c = x & 0x1f;
        x >>= 5;                                            // arithmetic shift, as pycocotools' signed long
        more = (c & 0x10) ? x != -1 : x != 0;
        ++n;
    }
    return n;
}

__device__ __forceinline__ unsigned char* rle_put(unsigned char* out, int x) {
    bool more = true;
    while (more) {
        int c = x & 0x1f;
        x >>= 5;
        more = (c & 0x10) ? x != -1 : x != 0;
        if (more) c |= 0x20;
        *out++ = (unsigned char)(c + 48);
    }
    return out;
}

struct SegmThreadState {
    int n, bytes, p0, p1, p2;        // scan state before the thread's chunk, string bytes before it
};

__device__ __forceinline__ void chunk_of(const SegmGeom& g, long long* e0, long long* e1) {
    const long long E = (long long)(g.x1 - g.x0) * (g.y1 - g.y0 + 1);
    const long long per = (E + kSegmThreads - 1) / kSegmThreads;
    *e0 = min((long long)threadIdx.x * per, E);
    *e1 = min(*e0 + per, E);
}

__global__ void __launch_bounds__(kSegmThreads)
segm_rle_sizes_kernel(const float* __restrict__ masks, const int* __restrict__ mask_class, const float* __restrict__ boxes, int Kc, int M,
                      int im_h, int im_w, float thresh, SegmThreadState* __restrict__ ws, int2* __restrict__ sizes) {
    using Scan = cub::BlockScan<Last3, kSegmThreads>;
    using Sum = cub::BlockScan<int, kSegmThreads>;
    __shared__ float pm[kSegmMaxS * kSegmMaxS];
    __shared__ union { typename Scan::TempStorage scan; typename Sum::TempStorage sum; } tmp;
    const int d = blockIdx.x, S = M + 2, N = im_h * im_w;
    load_padded(pm, masks, mask_class, d, Kc, M);
    const SegmGeom g = segm_geom(boxes + (size_t)d * 4, M, im_h, im_w);
    __syncthreads();
    long long e0, e1;
    chunk_of(g, &e0, &e1);
    Last3 mine{0, 0, 0, 0};
    segm_walk(pm, S, g, im_h, im_w, thresh, e0, e1, [&](int q) { push(mine, q); });
    Last3 before;
    Scan(tmp.scan).ExclusiveScan(mine, before, Last3{1, 0, 0, 0}, Last3Op());
    Last3 st = before;
    int bytes = 0, c;
    segm_walk(pm, S, g, im_h, im_w, thresh, e0, e1, [&](int q) { bytes += rle_len(rle_delta(st, q, &c)); push(st, q); });
    if (threadIdx.x == kSegmThreads - 1) bytes += rle_len(rle_delta(st, N, &c));     // st is now the whole detection's state
    __syncthreads();
    int bytes_before;
    Sum(tmp.sum).ExclusiveSum(bytes, bytes_before);
    ws[(size_t)d * kSegmThreads + threadIdx.x] = SegmThreadState{before.n, bytes_before, before.p0, before.p1, before.p2};
    if (threadIdx.x == kSegmThreads - 1) sizes[d] = make_int2(st.n, bytes_before + bytes);
}

__global__ void __launch_bounds__(kSegmThreads)
segm_rle_emit_kernel(const float* __restrict__ masks, const int* __restrict__ mask_class, const float* __restrict__ boxes, int D, int Kc,
                     int M, int im_h, int im_w, float thresh, const int2* __restrict__ sizes, const SegmThreadState* __restrict__ ws,
                     int* __restrict__ counts, long long* __restrict__ count_offs, unsigned char* __restrict__ strings,
                     long long* __restrict__ string_offs) {
    using Reduce = cub::BlockReduce<long long, kSegmThreads>;
    __shared__ float pm[kSegmMaxS * kSegmMaxS];
    __shared__ typename Reduce::TempStorage red;
    __shared__ long long offs[2];
    const int d = blockIdx.x, S = M + 2, N = im_h * im_w;
    load_padded(pm, masks, mask_class, d, Kc, M);
    const SegmGeom g = segm_geom(boxes + (size_t)d * 4, M, im_h, im_w);
    // this detection's offsets: the sizes of the detections before it
    long long co = 0, bo = 0;
    for (int i = threadIdx.x; i < d; i += kSegmThreads) { co += sizes[i].x; bo += sizes[i].y; }
    co = Reduce(red).Sum(co);
    __syncthreads();
    bo = Reduce(red).Sum(bo);
    if (threadIdx.x == 0) {
        offs[0] = co; offs[1] = bo;
        count_offs[d] = co; string_offs[d] = bo;
        if (d == D - 1) { count_offs[D] = co + sizes[d].x; string_offs[D] = bo + sizes[d].y; }
    }
    __syncthreads();
    const SegmThreadState s0 = ws[(size_t)d * kSegmThreads + threadIdx.x];
    Last3 st{s0.n, s0.p0, s0.p1, s0.p2};
    int* cnt = counts + offs[0];
    unsigned char* out = strings + offs[1] + s0.bytes;
    long long e0, e1;
    chunk_of(g, &e0, &e1);
    int c;
    segm_walk(pm, S, g, im_h, im_w, thresh, e0, e1, [&](int q) {
        const int x = rle_delta(st, q, &c);
        cnt[st.n - 1] = c;
        out = rle_put(out, x);
        push(st, q);
    });
    if (threadIdx.x == kSegmThreads - 1) {
        const int x = rle_delta(st, N, &c);
        cnt[st.n - 1] = c;
        rle_put(out, x);
    }
}

__global__ void __launch_bounds__(kSegmThreads)
paste_masks_kernel(const float* __restrict__ masks, const int* __restrict__ mask_class, const float* __restrict__ boxes, int Kc, int M,
                   int im_h, int im_w, float thresh, unsigned char* __restrict__ out) {
    __shared__ float pm[kSegmMaxS * kSegmMaxS];
    const int d = blockIdx.y, S = M + 2;
    const long long N = (long long)im_h * im_w;
    load_padded(pm, masks, mask_class, d, Kc, M);
    const SegmGeom g = segm_geom(boxes + (size_t)d * 4, M, im_h, im_w);
    __syncthreads();
    unsigned char* o = out + (size_t)d * N;
    for (long long p = (long long)blockIdx.x * kSegmThreads + threadIdx.x; p < N; p += (long long)gridDim.x * kSegmThreads) {
        const int y = (int)(p / im_w), x = (int)(p % im_w);
        const bool in = x >= g.x0 && x < g.x1 && y >= g.y0 && y < g.y1;
        o[p] = (in && segm_pixel(pm, S, g, x, y, thresh)) ? 1 : 0;
    }
}
}  // namespace

static bool segm_args_ok(int num_dets, int num_channels, int resolution, int im_h, int im_w) {
    return num_dets >= 0 && num_channels >= 1 && resolution >= 1 && resolution <= kSegmMaxM && im_h > 0 && im_w > 0 &&
           (long long)im_h * im_w < (1LL << 28);
}

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_segm_workspace_bytes(int num_dets) {
    if (num_dets <= 0) return 0;
    const size_t b = (size_t)num_dets * kSegmThreads * sizeof(SegmThreadState);
    return (b + 255) & ~(size_t)255;
}

int b200_segm_rle_sizes(const float* masks, const int* mask_class, const float* boxes, int D, int Kc, int M, int im_h, int im_w,
                        float thresh, int* sizes, void* ws, size_t workspace_bytes, b200_stream_t stream) {
    if (!segm_args_ok(D, Kc, M, im_h, im_w)) return B200_ROI_EINVAL;
    if (D == 0) return B200_ROI_OK;
    if (!masks || !mask_class || !boxes || !sizes) return B200_ROI_EINVAL;
    if (!ws || workspace_bytes < b200_segm_workspace_bytes(D)) return B200_ROI_EWORKSPACE;
    segm_rle_sizes_kernel<<<D, kSegmThreads, 0, stream>>>(masks, mask_class, boxes, Kc, M, im_h, im_w, thresh, (SegmThreadState*)ws,
                                                          (int2*)sizes);
    return finish_launch();
}

int b200_segm_rle_emit(const float* masks, const int* mask_class, const float* boxes, int D, int Kc, int M, int im_h, int im_w,
                       float thresh, const int* sizes, const void* ws, size_t workspace_bytes, int* counts, long long* count_offs,
                       unsigned char* strings, long long* string_offs, b200_stream_t stream) {
    if (!segm_args_ok(D, Kc, M, im_h, im_w)) return B200_ROI_EINVAL;
    if (D == 0) return B200_ROI_OK;
    if (!masks || !mask_class || !boxes || !sizes || !counts || !count_offs || !strings || !string_offs) return B200_ROI_EINVAL;
    if (!ws || workspace_bytes < b200_segm_workspace_bytes(D)) return B200_ROI_EWORKSPACE;
    segm_rle_emit_kernel<<<D, kSegmThreads, 0, stream>>>(masks, mask_class, boxes, D, Kc, M, im_h, im_w, thresh, (const int2*)sizes,
                                                         (const SegmThreadState*)ws, counts, count_offs, strings, string_offs);
    return finish_launch();
}

int b200_paste_masks(const float* masks, const int* mask_class, const float* boxes, int D, int Kc, int M, int im_h, int im_w, float thresh,
                     unsigned char* out, b200_stream_t stream) {
    if (!segm_args_ok(D, Kc, M, im_h, im_w) || D > 65535) return B200_ROI_EINVAL;
    if (D == 0) return B200_ROI_OK;
    if (!masks || !mask_class || !boxes || !out) return B200_ROI_EINVAL;
    const long long N = (long long)im_h * im_w;
    const long long blocks = (N + 8LL * kSegmThreads - 1) / (8LL * kSegmThreads);
    dim3 grid((unsigned)(blocks < 1024 ? blocks : 1024), D);
    paste_masks_kernel<<<grid, kSegmThreads, 0, stream>>>(masks, mask_class, boxes, Kc, M, im_h, im_w, thresh, out);
    return finish_launch();
}

}  // extern "C"
