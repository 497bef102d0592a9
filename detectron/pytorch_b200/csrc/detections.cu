// detections.cu -- test-time post-processing kernels of the detection head (SURVEY.md 8f N3):
//   soft-NMS      lib/utils/cython_nms.pyx:98-203 (reference), one warp per class problem
//   box voting    lib/utils/boxes.py:268-317 with cython_bbox.bbox_overlaps (lib/utils/cython_bbox.pyx:32-73)
// (classic per-class NMS is b200_nms_batched).  Problems are the per-class detection sets of one image, stored back to
// back; counts are launch geometry and come from the host.
#include "common.cuh"

namespace b200 {

namespace {
constexpr int kDetMaxProblems = 128;
struct DetBatch {
    int count;
    int n[kDetMaxProblems];
    int off[kDetMaxProblems];
};

// Soft-NMS exactly as the reference runs it: for i = 0 .. N-1: move the best remaining box to slot i (first maximum
// wins), decay the scores of the boxes behind it by their overlap with it, and drop boxes whose score fell below the
// threshold by overwriting them with the current last box (N shrinks; the moved box is examined in place).  The score
// updates are independent per box and run across the lanes; the drop pass depends on the running N and runs on lane 0.
// method: 1 linear, 2 gaussian, else hard.  boxes: (n, 5) rows, modified in place; inds: original row indices.
__global__ void __launch_bounds__(32)
soft_nms_kernel(float* __restrict__ boxes_all, int* __restrict__ inds_all, int* __restrict__ n_out, const __grid_constant__ DetBatch db,
                float sigma, float Nt, float threshold, int method) {
    const int p = blockIdx.x, lane = threadIdx.x;
    float* boxes = boxes_all + (size_t)db.off[p] * 5;
    int* inds = inds_all + db.off[p];
    int N = db.n[p];
    for (int k = lane; k < N; k += 32) inds[k] = k;
    __syncwarp();
    for (int i = 0; i < N; ++i) {
        // best remaining box: maximum score, first index among equals (the reference scans with `maxscore < score`)
        float best = -INFINITY; int bpos = 0x7fffffff;
        for (int k = i + lane; k < N; k += 32) {
            const float s = boxes[k * 5 + 4];
            if (s > best) { best = s; bpos = k; }                   // ascending k per lane: first maximum of the lane
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int op = __shfl_xor_sync(0xffffffffu, bpos, o);
            if (ob > best || (ob == best && op < bpos)) { best = ob; bpos = op; }
        }
        const int maxpos = (bpos == 0x7fffffff) ? i : bpos;
        __syncwarp();
        if (lane < 5) {                                             // swap rows i and maxpos (and their indices)
            const float a = boxes[i * 5 + lane], b = boxes[maxpos * 5 + lane];
            boxes[i * 5 + lane] = b; boxes[maxpos * 5 + lane] = a;
        } else if (lane == 5) {
            const int a = inds[i], b = inds[maxpos];
            inds[i] = b; inds[maxpos] = a;
        }
        __syncwarp();
        const float tx1 = boxes[i * 5], ty1 = boxes[i * 5 + 1], tx2 = boxes[i * 5 + 2], ty2 = boxes[i * 5 + 3];
        // The C that Cython generates from the .pyx adds the literal 1.0 in double: a box's area is a double product rounded
        // to float once (cython_area), iw / ih are double sums rounded to float, and the union is the double expression
        // (t_area + area) - iw * ih rounded to float once.  The intersection, the IoU and the score product are float.
        const double t_area = __dmul_rn(__dadd_rn((double)__fsub_rn(tx2, tx1), 1.0), __dadd_rn((double)__fsub_rn(ty2, ty1), 1.0));
        for (int k = i + 1 + lane; k < N; k += 32) {
            const float x1 = boxes[k * 5], y1 = boxes[k * 5 + 1], x2 = boxes[k * 5 + 2], y2 = boxes[k * 5 + 3];
            const float area = cython_area(x1, y1, x2, y2);
            const float iw = (float)__dadd_rn((double)__fsub_rn(fminf(tx2, x2), fmaxf(tx1, x1)), 1.0);
            if (iw > 0.f) {
                const float ih = (float)__dadd_rn((double)__fsub_rn(fminf(ty2, y2), fmaxf(ty1, y1)), 1.0);
                if (ih > 0.f) {
                    const float inter = __fmul_rn(iw, ih);
                    const float ua = (float)__dsub_rn(__dadd_rn(t_area, (double)area), (double)inter);
                    const float ov = __fdiv_rn(inter, ua);
                    float weight;
                    if (method == 1) weight = (ov > Nt) ? __fsub_rn(1.f, ov) : 1.f;
                    else if (method == 2) weight = (float)exp((double)__fdiv_rn(-__fmul_rn(ov, ov), sigma));   // float argument, np.exp in double
                    else weight = (ov > Nt) ? 0.f : 1.f;
                    const float ns = __fmul_rn(weight, boxes[k * 5 + 4]);
                    boxes[k * 5 + 4] = ns;
                    if (ns < threshold) inds[k] = ~inds[k];          // drop candidate (the reference only tests boxes that overlap)
                }
            }
        }
        __syncwarp();
        if (lane == 0) {                                            // drop pass, in the reference's order
            int pos = i + 1;
            while (pos < N) {
                if (inds[pos] < 0) {
                    for (int c = 0; c < 5; ++c) boxes[pos * 5 + c] = boxes[(N - 1) * 5 + c];
                    inds[pos] = inds[N - 1];                        // the moved box keeps its own mark and is examined in place
                    --N;
                } else {
                    ++pos;
                }
            }
        }
        N = __shfl_sync(0xffffffffu, N, 0);
        __syncwarp();
    }
    if (lane == 0) n_out[p] = N;
}

// Box voting: every kept detection becomes the score-weighted average of all detections of its class that overlap it
// by at least `thresh` (bbox_overlaps convention: +1 on widths / heights, IoU in fp32).  One thread per kept detection.
// scoring: 0 ID, 1 AVG, 2 IOU_AVG, 3 TEMP_AVG, 4 GENERALIZED_AVG, 5 QUASI_SUM (lib/utils/boxes.py:283-312).
__global__ void __launch_bounds__(128)
box_voting_kernel(const float* __restrict__ top_all, const float* __restrict__ all_all, float* __restrict__ out_all,
                  const __grid_constant__ DetBatch top_b, const __grid_constant__ DetBatch all_b, float thresh, int scoring, float beta) {
    const int p = blockIdx.y;
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= top_b.n[p]) return;
    const float* top = top_all + (size_t)(top_b.off[p] + k) * 5;
    const float* all = all_all + (size_t)all_b.off[p] * 5;
    float* out = out_all + (size_t)(top_b.off[p] + k) * 5;
    const int n = all_b.n[p];
    const float bx1 = top[0], by1 = top[1], bx2 = top[2], by2 = top[3];
    double sx1 = 0, sy1 = 0, sx2 = 0, sy2 = 0, sw = 0, s_temp = 0, s_iou_w = 0, s_iou_p = 0, s_gen = 0;
    int cnt = 0;
    for (int j = 0; j < n; ++j) {
        const float qx1 = all[j * 5], qy1 = all[j * 5 + 1], qx2 = all[j * 5 + 2], qy2 = all[j * 5 + 3], w = all[j * 5 + 4];
        // utils.boxes.box_voting: bbox_overlaps(top_boxes, all_boxes) -> the kept detection is the "boxes" row
        const float ov = cython_iou(bx1, by1, bx2, by2, qx1, qy1, qx2, qy2, cython_area(qx1, qy1, qx2, qy2));
        if (ov >= thresh) {
            sx1 += (double)w * qx1; sy1 += (double)w * qy1; sx2 += (double)w * qx2; sy2 += (double)w * qy2; sw += w;
            ++cnt;
            if (scoring == 2) { s_iou_w += ov; s_iou_p += (double)ov * w; }
            else if (scoring == 3) {                                   // softmax over (w, 1 - w) with temperature beta
                const double a = w, b = 1.0 - (double)w, m = a > b ? a : b;
                const double ea = exp(log(a / m) / beta), eb = exp(log(b / m) / beta);
                s_temp += ea / (ea + eb);
            } else if (scoring == 4) s_gen += pow((double)w, (double)beta);
        }
    }
    out[0] = (float)(sx1 / sw); out[1] = (float)(sy1 / sw); out[2] = (float)(sx2 / sw); out[3] = (float)(sy2 / sw);
    float score = top[4];
    if (cnt > 0) {
        if (scoring == 1) score = (float)(sw / cnt);
        else if (scoring == 2) score = (float)(s_iou_p / s_iou_w);
        else if (scoring == 3) score = (float)(s_temp / cnt);
        else if (scoring == 4) score = (float)pow(s_gen / cnt, 1.0 / (double)beta);
        else if (scoring == 5) score = (float)(sw / pow((double)cnt, (double)beta));
    }
    out[4] = score;
}

bool det_batch(const int* counts, int num, DetBatch* b, long long* total) {
    if (num < 1 || num > kDetMaxProblems) return false;
    long long off = 0;
    b->count = num;
    for (int p = 0; p < kDetMaxProblems; ++p) {
        const int n = p < num ? counts[p] : 0;
        if (n < 0) return false;
        b->n[p] = n; b->off[p] = (int)off; off += n;
        if (off > 0x7fffffffLL) return false;
    }
    *total = off;
    return true;
}
}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

int b200_soft_nms_batched(float* boxes, const int* counts, int num, float sigma, float Nt, float threshold, int method, int* inds,
                          int* n_out, b200_stream_t stream) {
    if (!counts || num < 1 || !n_out) return B200_ROI_EINVAL;
    long long total = 0;
    for (int p = 0; p < num && p < 128; ++p) total += counts[p] > 0 ? counts[p] : 0;
    if (total > 0 && (!boxes || !inds)) return B200_ROI_EINVAL;
    DetBatch b;
    if (!det_batch(counts, num, &b, &total)) return B200_ROI_EINVAL;
    soft_nms_kernel<<<num, 32, 0, stream>>>(boxes, inds, n_out, b, sigma, Nt, threshold, method);
    return finish_launch();
}

int b200_box_voting_batched(const float* top, const int* top_counts, const float* all, const int* all_counts, int num, float thresh,
                            int scoring, float beta, float* out, b200_stream_t stream) {
    if (!top_counts || !all_counts || num < 1) return B200_ROI_EINVAL;
    long long total = 0;
    for (int p = 0; p < num && p < 128; ++p) total += top_counts[p] > 0 ? top_counts[p] : 0;
    if (total > 0 && (!top || !all || !out)) return B200_ROI_EINVAL;
    if (scoring < 0 || scoring > 5) return B200_ROI_EINVAL;
    DetBatch tb, ab; long long t1 = 0, t2 = 0;
    if (!det_batch(top_counts, num, &tb, &t1) || !det_batch(all_counts, num, &ab, &t2)) return B200_ROI_EINVAL;
    int mx = 0;
    for (int p = 0; p < num; ++p) mx = top_counts[p] > mx ? top_counts[p] : mx;
    if (mx == 0) return B200_ROI_OK;
    dim3 grid((mx + 127) / 128, num);
    box_voting_kernel<<<grid, 128, 0, stream>>>(top, all, out, tb, ab, thresh, scoring, beta);
    return finish_launch();
}

}  // extern "C"
