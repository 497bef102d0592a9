// mask_targets.cu -- Mask R-CNN training mask targets on the device (the training-time add_mask_rcnn_blobs).
//
// The reference does this on the host, per image, inside the model's forward:
//   lib/roi_data/mask_rcnn.py:34-48       non-crowd objects with a class, their tight polygon boxes (utils/segms.py:120-131)
//   lib/roi_data/mask_rcnn.py:50-76       cython_bbox IoU of every fg RoI against those boxes, first argmax, and one
//                                         rasterisation per RoI (utils/segms.py:93-117: float32 normalisation to the RoI,
//                                         pycocotools frPyObjects + decode at M x M, union of the object's polygons)
//   lib/roi_data/mask_rcnn.py:77-122      the empty-fg fallback and the class-specific (R, K * M * M) int32 expansion
// All images of a step go through the same two launches:
//   mask_boxes_kernel     one warp per object: tight box of its polygons
//   mask_targets_kernel   one CTA per RoI: argmax, rasterisation, the whole output row with 16-byte stores
//
// The rasteriser is pycocotools' rleFrPoly + rleDecode (oracle/masks.py restates it), bit for bit, but its work per edge is
// bounded by the M columns the edge can cross rather than by its upsampled length: along an edge the upsampled column u is
// monotone, so the single walk step that crosses column c (u from 5c + 2 to 5c + 3 or back) is found by bisection with the
// reference's own rounding.  Crossings toggle one bit of a per-column 64-bit word (XOR, so duplicates cancel); a prefix
// parity over the column-major order, carried across columns, gives the filled polygon.
#include "poly_walk.cuh"

namespace b200 {

constexpr int kMaskMaxImages = 64;
constexpr int kMaskMaxM = 64;

namespace {

constexpr int kMaskThreads = 256;
constexpr int kPolyBatch = 16;       // polygons rasterised side by side in one CTA (an object with more takes several rounds)

struct MaskImages {
    int num_images;
    int obj_begin[kMaskMaxImages + 1];
};

// the tight box of each object's polygons (segms.py:120-131); float32 min / max equal the float64 ones, rounded
__global__ void __launch_bounds__(kMaskThreads)
mask_boxes_kernel(int num_objects, int num_polys, int num_coords, const int* __restrict__ poly_begin, const int* __restrict__ coord_begin,
                  const float* __restrict__ coords, float4* __restrict__ boxes) {
    const int o = blockIdx.x * (kMaskThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (o >= num_objects) return;
    const int p0 = min(max(__ldg(poly_begin + o), 0), num_polys), p1 = min(max(__ldg(poly_begin + o + 1), p0), num_polys);
    const int c0 = min(max(__ldg(coord_begin + p0), 0), num_coords), c1 = min(max(__ldg(coord_begin + p1), c0), num_coords);
    float x0 = INFINITY, y0 = INFINITY, x1 = -INFINITY, y1 = -INFINITY;
    for (int i = c0 + 2 * lane; i + 1 < c1; i += 64) {                  // polygons start at even offsets
        const float x = __ldg(coords + i), y = __ldg(coords + i + 1);
        x0 = fminf(x0, x); x1 = fmaxf(x1, x); y0 = fminf(y0, y); y1 = fmaxf(y1, y);
    }
    for (int s = 16; s > 0; s >>= 1) {
        x0 = fminf(x0, __shfl_xor_sync(0xffffffffu, x0, s)); y0 = fminf(y0, __shfl_xor_sync(0xffffffffu, y0, s));
        x1 = fmaxf(x1, __shfl_xor_sync(0xffffffffu, x1, s)); y1 = fmaxf(y1, __shfl_xor_sync(0xffffffffu, y1, s));
    }
    if (lane == 0) boxes[o] = make_float4(x0, y0, x1, y1);
}

using poly::Edge;
using poly::edge_u;
using poly::edge_v;
using poly::make_edge;
using poly::kUpsample;

// a kept crossing toggles bit yd of column word xd (yd == h is the top of the next column; past the last column it is the
// sentinel)
__device__ __forceinline__ void crossing(int pu, int pv, int qu, int qv, int h, int w, unsigned long long* tog) {
    int c, y;
    if (!poly::crossing(pu, pv, qu, qv, h, w, c, y)) return;
    if (y == h) { ++c; y = 0; }
    if (c < w) atomicXor(tog + c, 1ull << y);
}

__device__ __forceinline__ void edge_crossings(const Edge& e, int h, int w, unsigned long long* tog) {
    poly::edge_crossings(e, w, [&](int pu, int pv, int qu, int qv) { crossing(pu, pv, qu, qv, h, w, tog); });
}

// float32 normalisation to the RoI (segms.py:104-110), then rleFrPoly's (int)(5 * x + .5)
__device__ __forceinline__ int2 upsampled_vertex(const float* __restrict__ xy, float4 box, float fM, float bw, float bh) {
    const float x = __fdiv_rn(__fmul_rn(__fsub_rn(__ldg(xy), box.x), fM), bw);
    const float y = __fdiv_rn(__fmul_rn(__fsub_rn(__ldg(xy + 1), box.y), fM), bh);
    return make_int2(__double2int_rz(__dadd_rn(__dmul_rn((double)kUpsample, (double)x), 0.5)),
                     __double2int_rz(__dadd_rn(__dmul_rn((double)kUpsample, (double)y), 0.5)));
}

__global__ void __launch_bounds__(kMaskThreads)
mask_targets_kernel(const __grid_constant__ MaskImages im, const float4* __restrict__ rois, const int* __restrict__ roi_image,
                    const int* __restrict__ roi_class, int num_objects, int num_polys, int num_coords, const int* __restrict__ poly_begin,
                    const int* __restrict__ coord_begin, const float* __restrict__ coords, const float4* __restrict__ boxes, int M,
                    int num_classes, long long row_len, int* __restrict__ out) {
    __shared__ unsigned long long s_tog[kPolyBatch][kMaskMaxM];
    __shared__ unsigned long long s_mask[kMaskMaxM];
    __shared__ int s_cb[kPolyBatch + 1];
    __shared__ unsigned long long s_best[kMaskThreads / 32];
    const int r = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int n = __ldg(roi_image + r), cls = __ldg(roi_class + r);
    const int o0 = (n >= 0 && n < im.num_images) ? im.obj_begin[n] : 0, o1 = (n >= 0 && n < im.num_images) ? im.obj_begin[n + 1] : 0;
    const bool has_mask = cls > 0 && o1 > o0 && (num_classes == 0 || cls < num_classes);
    for (int i = t; i < kPolyBatch * kMaskMaxM; i += kMaskThreads) (&s_tog[0][0])[i] = 0ull;
    if (t < kMaskMaxM) s_mask[t] = 0ull;
    if (has_mask) {
        // first argmax of the IoU against the image's object boxes (mask_rcnn.py:57-64): key = IoU bits (>= 0) | ~index
        const float4 b = __ldg(rois + r);
        unsigned long long best = 0ull;
        for (int j = o0 + t; j < o1; j += kMaskThreads) {
            const float4 q = __ldg(boxes + j);
            const float iou = cython_iou(b.x, b.y, b.z, b.w, q.x, q.y, q.z, q.w, cython_area(q.x, q.y, q.z, q.w));
            const unsigned long long key = ((unsigned long long)__float_as_uint(iou) << 32) | (unsigned)(~(j - o0));
            best = key > best ? key : best;
        }
        for (int s = 16; s > 0; s >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, s);
            best = other > best ? other : best;
        }
        if (lane == 0) s_best[warp] = best;
        __syncthreads();
        best = s_best[0];
        for (int w = 1; w < kMaskThreads / 32; ++w) best = s_best[w] > best ? s_best[w] : best;
        const int obj = o0 + (int)(~(unsigned)(best & 0xffffffffull));
        const int p0 = min(max(__ldg(poly_begin + obj), 0), num_polys), p1 = min(max(__ldg(poly_begin + obj + 1), p0), num_polys);
        const float fM = (float)M, bw = fmaxf(__fsub_rn(b.z, b.x), 1.f), bh = fmaxf(__fsub_rn(b.w, b.y), 1.f);
        for (int pb = p0; pb < p1; pb += kPolyBatch) {
            const int np = min(kPolyBatch, p1 - pb);
            if (t <= np) s_cb[t] = min(max(__ldg(coord_begin + pb + t), 0), num_coords) & ~1;
            __syncthreads();
            const int v0 = s_cb[0] >> 1, nv = (s_cb[np] >> 1) - v0;
            for (int i = t; i < nv; i += kMaskThreads) {                 // one thread per edge: vertex g -> its successor in the ring
                const int g = v0 + i;
                int p = 0;
                while (p + 1 < np && 2 * g >= s_cb[p + 1]) ++p;
                const int pv0 = s_cb[p] >> 1, k = (s_cb[p + 1] >> 1) - pv0, j = g - pv0;
                if (k < 1) continue;
                const float* base = coords + 2 * pv0;
                const int2 a = upsampled_vertex(base + 2 * j, b, fM, bw, bh);
                const int2 c = upsampled_vertex(base + 2 * ((j + 1) % k), b, fM, bw, bh);
                const Edge e = make_edge(a.x, a.y, c.x, c.y);
                edge_crossings(e, M, M, s_tog[p]);
                if (j > 0) {                                             // the step from the previous edge's last point
                    const int2 z = upsampled_vertex(base + 2 * (j - 1), b, fM, bw, bh);
                    const Edge f = make_edge(z.x, z.y, a.x, a.y);
                    crossing(edge_u(f, f.n), edge_v(f, f.n), edge_u(e, 0), edge_v(e, 0), M, M, s_tog[p]);
                }
            }
            __syncthreads();
            // fill: pixel (x, y) = parity of the toggles at column-major positions <= x * M + y; union over the polygons
            const unsigned long long hmask = M == 64 ? ~0ull : ((1ull << M) - 1ull);
            for (int p = warp; p < np; p += kMaskThreads / 32) {
                unsigned long long w0 = lane < M ? s_tog[p][lane] : 0ull, w1 = lane + 32 < M ? s_tog[p][lane + 32] : 0ull;
                const unsigned b0 = __ballot_sync(0xffffffffu, __popcll(w0) & 1), b1 = __ballot_sync(0xffffffffu, __popcll(w1) & 1);
                const unsigned below = (1u << lane) - 1u;
                const unsigned carry0 = __popc(b0 & below) & 1, carry1 = (__popc(b0) + __popc(b1 & below)) & 1;
#pragma unroll
                for (int s = 1; s < 64; s <<= 1) { w0 ^= w0 << s; w1 ^= w1 << s; }
                if (lane < M) { atomicOr(s_mask + lane, (carry0 ? ~w0 : w0) & hmask); s_tog[p][lane] = 0ull; }
                if (lane + 32 < M) { atomicOr(s_mask + lane + 32, (carry1 ? ~w1 : w1) & hmask); s_tog[p][lane + 32] = 0ull; }
            }
            __syncthreads();
        }
    }
    __syncthreads();
    // the row: the class slice (the whole row when class-agnostic) holds the mask, -1 everywhere else (mask_rcnn.py:108-122)
    const int MM = M * M;
    const long long s0 = has_mask ? (num_classes > 0 ? (long long)cls * MM : 0) : row_len;
    int* row = out + (long long)r * row_len;
    auto value = [&](long long i) -> int {
        if (i < s0 || i >= s0 + MM) return -1;
        const int q = (int)(i - s0), y = q / M, x = q - y * M;
        return (int)((s_mask[x] >> y) & 1ull);
    };
    if ((row_len & 3) == 0) {
        int4* row4 = reinterpret_cast<int4*>(row);
        for (long long i = t; i < row_len / 4; i += kMaskThreads) {
            const long long e = 4 * i;
            row4[i] = (e + 4 <= s0 || e >= s0 + MM) ? make_int4(-1, -1, -1, -1) : make_int4(value(e), value(e + 1), value(e + 2), value(e + 3));
        }
    } else {
        for (long long i = t; i < row_len; i += kMaskThreads) row[i] = value(i);
    }
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_mask_targets(const float* rois, const int* roi_image, const int* roi_class, int num_rois, int num_images, const int* obj_begin,
                      int num_polys, const int* poly_begin, int num_coords, const int* coord_begin, const float* coords, int M, int num_classes,
                      float* obj_boxes, int* masks_out, b200_stream_t stream) {
    if (!rois || !roi_image || !roi_class || !obj_begin || !poly_begin || !coord_begin || !coords || !obj_boxes || !masks_out)
        return B200_ROI_EINVAL;
    if (num_rois < 1 || num_images < 1 || num_images > kMaskMaxImages || M < 1 || M > kMaskMaxM || num_classes < 0 ||
        num_polys < 0 || num_coords < 0 || (num_coords & 1))
        return B200_ROI_EINVAL;
    MaskImages im{};
    im.num_images = num_images;
    if (obj_begin[0] != 0) return B200_ROI_EINVAL;
    for (int i = 0; i <= num_images; ++i) {
        if (i > 0 && obj_begin[i] < obj_begin[i - 1]) return B200_ROI_EINVAL;
        im.obj_begin[i] = obj_begin[i];
    }
    const int num_objects = obj_begin[num_images];
    if (num_objects > num_polys) return B200_ROI_EINVAL;                // every object has at least one polygon
    const long long row_len = (long long)(num_classes > 0 ? num_classes : 1) * M * M;
    if (row_len > (1LL << 31) || (long long)num_rois * row_len > (1LL << 40)) return B200_ROI_EINVAL;
    if ((row_len & 3) == 0 && ((uintptr_t)masks_out & 15)) return B200_ROI_EINVAL;   // the 16-byte stores need an aligned blob
    if ((uintptr_t)rois & 15 || (uintptr_t)obj_boxes & 15) return B200_ROI_EINVAL;
    mask_boxes_kernel<<<max((num_objects + kMaskThreads / 32 - 1) / (kMaskThreads / 32), 1), kMaskThreads, 0, stream>>>(
        num_objects, num_polys, num_coords, poly_begin, coord_begin, coords, (float4*)obj_boxes);
    mask_targets_kernel<<<num_rois, kMaskThreads, 0, stream>>>(im, (const float4*)rois, roi_image, roi_class, num_objects, num_polys,
                                                               num_coords, poly_begin, coord_begin, coords, (const float4*)obj_boxes, M,
                                                               num_classes, row_len, masks_out);
    return finish_launch(2);
}

}  // extern "C"
