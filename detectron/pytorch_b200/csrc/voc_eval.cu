// voc_eval.cu -- PASCAL VOC detection matching on the device (the per-detection loop of the reference's voc_eval; oracle/voc_eval.py
// restates it).
//
// Detections of every class are packed into one array; within a class they are in rank order (descending score, ties in file order),
// so a detection's index is its rank.  Ground truth is stored per (class, image) pair as one contiguous row range (CSR).
//   voc_overlap_kernel  one thread per detection: IoU against the pair's ground truth, ovmax / jmax as numpy's max / argmax give
//                       them; a qualifying detection (ovmax > ovthresh, jmax not difficult) claims jmax with atomicMin(rank)
//   voc_outcome_kernel  one thread per qualifying detection: it is the tp when its claim won, otherwise a duplicate (fp)
// The claims do not depend on each other: a ground-truth box's tp is the lowest-ranked detection that qualifies for it, which is the
// first one the reference's sequential loop reaches.  Every float64 step is an _rn intrinsic so no contraction changes a rounding.
#include <cstdint>

#include "common.cuh"

namespace b200 {

namespace {

constexpr int kVocThreads = 256;
constexpr unsigned char kFp = 0, kTp = 1, kNeither = 2, kCandidate = 3;

// np.maximum / np.minimum: a NaN operand gives NaN
__device__ __forceinline__ double np_max(double a, double b) { return (isnan(a) || a >= b) ? a : b; }
__device__ __forceinline__ double np_min(double a, double b) { return (isnan(a) || a <= b) ? a : b; }

// The reference's overlaps row for box b against ground truth g0 .. g1 - 1, reduced to jmax (numpy's argmax: the first maximum, or the
// first NaN, which also makes ovmax NaN).  Returns -1 without ground truth (ovmax = -inf); *qualifies = ovmax > ovthresh.
__device__ __forceinline__ int best_overlap(double4 b, const double4* __restrict__ gt, int g0, int g1, double ovthresh, bool* qualifies) {
    const double bw = __dadd_rn(__dsub_rn(b.z, b.x), 1.0), bh = __dadd_rn(__dsub_rn(b.w, b.y), 1.0);
    const double barea = __dmul_rn(bw, bh);
    double ovmax = -INFINITY;
    int jmax = -1;
    for (int g = g0; g < g1; ++g) {
        const double4 q = gt[g];
        const double iw = np_max(__dadd_rn(__dsub_rn(np_min(q.z, b.z), np_max(q.x, b.x)), 1.0), 0.0);
        const double ih = np_max(__dadd_rn(__dsub_rn(np_min(q.w, b.w), np_max(q.y, b.y)), 1.0), 0.0);
        const double inters = __dmul_rn(iw, ih);
        const double garea = __dmul_rn(__dadd_rn(__dsub_rn(q.z, q.x), 1.0), __dadd_rn(__dsub_rn(q.w, q.y), 1.0));
        const double ov = __ddiv_rn(inters, __dsub_rn(__dadd_rn(barea, garea), inters));
        if (isnan(ov)) { ovmax = ov; jmax = g; break; }
        if (jmax < 0 || ov > ovmax) { ovmax = ov; jmax = g; }
    }
    *qualifies = ovmax > ovthresh;
    return jmax;
}

__global__ void __launch_bounds__(kVocThreads)
voc_overlap_kernel(int num_dets, double ovthresh, const int* __restrict__ pair_gt_begin, const double4* __restrict__ gt_box,
                   const unsigned char* __restrict__ gt_difficult, const int* __restrict__ det_pair, const double4* __restrict__ det_box,
                   unsigned* __restrict__ first_rank, unsigned char* __restrict__ outcome) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= num_dets) return;
    const int p = det_pair[d];
    bool qualifies;
    const int j = best_overlap(det_box[d], gt_box, pair_gt_begin[p], pair_gt_begin[p + 1], ovthresh, &qualifies);
    unsigned char o = kFp;
    if (qualifies) {
        if (gt_difficult[j]) {
            o = kNeither;
        } else {
            atomicMin(first_rank + j, (unsigned)d);
            o = kCandidate;
        }
    }
    outcome[d] = o;
}

__global__ void __launch_bounds__(kVocThreads)
voc_outcome_kernel(int num_dets, double ovthresh, const int* __restrict__ pair_gt_begin, const double4* __restrict__ gt_box,
                   const int* __restrict__ det_pair, const double4* __restrict__ det_box, const unsigned* __restrict__ first_rank,
                   unsigned char* __restrict__ outcome) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= num_dets || outcome[d] != kCandidate) return;
    const int p = det_pair[d];
    bool qualifies;
    const int j = best_overlap(det_box[d], gt_box, pair_gt_begin[p], pair_gt_begin[p + 1], ovthresh, &qualifies);
    outcome[d] = first_rank[j] == (unsigned)d ? kTp : kFp;
}

}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_voc_match(int num_dets, int num_pairs, int num_gt, double ovthresh, const int* pair_gt_begin, const double* gt_box,
                   const unsigned char* gt_difficult, const int* det_pair, const double* det_box, int* workspace, unsigned char* outcome,
                   b200_stream_t stream) {
    if (num_dets < 0 || num_pairs < 0 || num_gt < 0 || (num_dets > 0 && num_pairs == 0)) return B200_ROI_EINVAL;
    if (num_gt > 0 && (!gt_box || !gt_difficult || !workspace)) return B200_ROI_EINVAL;
    if (num_dets > 0 && (!pair_gt_begin || !det_pair || !det_box || !outcome)) return B200_ROI_EINVAL;
    if (((uintptr_t)gt_box | (uintptr_t)det_box) & 15) return B200_ROI_EINVAL;
    if (num_dets == 0) return B200_ROI_OK;
    unsigned* first_rank = (unsigned*)workspace;                         // all ones: no claim yet
    int launches = 0;
    if (num_gt > 0) {
        if (cudaMemsetAsync(workspace, 0xff, (size_t)num_gt * sizeof(unsigned), stream) != cudaSuccess) return finish_launch(0);
    }
    const int grid = (num_dets + kVocThreads - 1) / kVocThreads;
    voc_overlap_kernel<<<grid, kVocThreads, 0, stream>>>(num_dets, ovthresh, pair_gt_begin, (const double4*)gt_box, gt_difficult, det_pair,
                                                         (const double4*)det_box, first_rank, outcome);
    ++launches;
    if (num_gt > 0) {
        voc_outcome_kernel<<<grid, kVocThreads, 0, stream>>>(num_dets, ovthresh, pair_gt_begin, (const double4*)gt_box, det_pair,
                                                             (const double4*)det_box, first_rank, outcome);
        ++launches;
    }
    return finish_launch(launches);
}

}  // extern "C"
