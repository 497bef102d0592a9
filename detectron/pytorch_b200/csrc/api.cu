// api.cu -- the extern "C" boundary of libb200_roi_ops.so (see include/b200_roi_ops.h).
// Argument validation + dispatch only; kernels live in the per-op translation units.
#include "common.cuh"
#include <mutex>
#include <stdlib.h>
#include <string.h>

namespace b200 {
unsigned long long g_launch_count = 0;

static const char* const kOptionNames[kNumOptions] = {"B200_ROI_ALIGN_PATH", "B200_ROI_ALIGN_BWD_PATH", "B200_ROI_ALIGN_BWD_CPL",
                                                      "B200_NMS_SCAN"};
static int g_options[kNumOptions];
static std::once_flag g_options_once;

static void options_init() {
    for (int i = 0; i < kNumOptions; ++i) {
        const char* e = getenv(kOptionNames[i]);
        __atomic_store_n(&g_options[i], e ? (int)(unsigned char)e[0] : 0, __ATOMIC_RELAXED);
    }
}

int option_get(Option which) {
    std::call_once(g_options_once, options_init);
    return __atomic_load_n(&g_options[which], __ATOMIC_RELAXED);
}

static int option_set(const char* name, const char* value) {
    std::call_once(g_options_once, options_init);
    if (!name) return B200_ROI_EINVAL;
    for (int i = 0; i < kNumOptions; ++i)
        if (strcmp(name, kOptionNames[i]) == 0) {
            __atomic_store_n(&g_options[i], value ? (int)(unsigned char)value[0] : 0, __ATOMIC_RELAXED);
            return B200_ROI_OK;
        }
    return B200_ROI_EINVAL;
}

int roi_align_forward_generic(const float*, float, int, int, int, int, int, int, int, int, const float*, float*, const int*, cudaStream_t);
int roi_align_backward_generic(const float*, float, int, int, int, int, int, int, int, int, const float*, float*, const int*, cudaStream_t);
int roi_align_legacy_forward(const float*, float, int, int, int, int, int, int, int, const float*, float*, cudaStream_t);
int roi_align_legacy_backward(const float*, float, int, int, int, int, int, int, int, const float*, float*, cudaStream_t);
int roi_pool_forward(const float*, float, int, int, int, int, int, int, int, const float*, float*, int*, cudaStream_t);
int roi_pool_backward(const float*, float, int, int, int, int, int, int, int, const float*, float*, const int*, cudaStream_t);
int roi_crop_forward(const float*, const float*, int, int, int, int, int, int, int, float*, cudaStream_t);
int roi_crop_backward(const float*, const float*, int, int, int, int, int, int, int, float*, float*, void*, size_t, cudaStream_t);
size_t roi_crop_backward_workspace_bytes(int, int, int, int, int, int, int);
size_t nms_workspace_bytes(int);
int proposal_decode(const float*, const float*, const long long*, const float*, int, int, int, int, float, float, float, float, float*, int*, cudaStream_t);
size_t roi_align_tiled_workspace_bytes(int, int, int, int, int, int, int);
void nms_set_timing_buffer(unsigned long long*);
void roi_align_stream_set_debug_buffer(unsigned long long*);
int roi_align_forward_tiled(const float*, float, int, int, int, int, int, int, int, int, const float*, float*, const int*, void*, size_t, cudaStream_t);
size_t roi_align_stream_workspace_bytes(int, int, int, int, int, int, int);
int roi_align_forward_stream(const float*, float, int, int, int, int, int, int, int, int, const float*, float*, const int*, void*, size_t, cudaStream_t);
size_t roi_align_strip_workspace_bytes(int, int, int, int, int, int, int);
size_t roi_align_strip_fpn_workspace_bytes(int, const int*, const int*, int, int, int, int, int);
int roi_align_forward_strip_fpn(int, const float* const*, const int*, const int*, const float*, const int*, int, int, int, int, int, int,
                                const float*, float*, const int*, void*, size_t, cudaStream_t);
int roi_align_forward_strip(const float*, float, int, int, int, int, int, int, int, int, const float*, float*, const int*, void*, size_t, cudaStream_t);
void roi_align_strip_set_debug_buffer(unsigned long long*);

size_t topk_batched_workspace_bytes(int);
int topk_batched(const float* const*, const int*, const int*, const int*, int, long long*, float*, void*, size_t, cudaStream_t);
int bbox_overlaps(const float*, int, const float*, int, float*, cudaStream_t);
int roi_assign(const float*, int, const float*, const int*, int, float*, int*, int*, cudaStream_t);
int roi_select(const float*, int, float, float, float, int*, int*, int*, cudaStream_t);
int fast_rcnn_targets(const float*, const float*, const int*, const int*, const int*, int, int, const float*, int, int, float, float, int*,
                      float*, float*, float*, float*, cudaStream_t);
size_t segm_workspace_bytes(int);
bool segm_args_ok(int, int, int, int, int);
int segm_rle_sizes(const float*, const int*, const float*, int, int, int, int, int, float, int*, void*, cudaStream_t);
int segm_rle_emit(const float*, const int*, const float*, int, int, int, int, int, float, const int*, const void*, int*, long long*,
                  unsigned char*, long long*, cudaStream_t);
int paste_masks(const float*, const int*, const float*, int, int, int, int, int, float, unsigned char*, cudaStream_t);
bool keypoints_args_ok(int, int, int, int);
bool nms_oks_args_ok(int, int);
int heatmaps_to_keypoints(const float*, const float*, int, int, int, int, float*, cudaStream_t);
int nms_oks(const float*, const float*, int, double, int*, int*, cudaStream_t);
int rpn_total_anchors(int, const int*, const int*);
size_t rpn_workspace_bytes(int, int, int);
int rpn_labels(int, const int*, const int*, const double*, const double*, int, const double*, const int*, const float*, double, float, float,
               int*, void*, size_t, cudaStream_t);
int rpn_emit(int, const int*, const int*, const double*, const double*, int, const double*, const int*, const float*, double, const int*,
             const int*, const int*, const int*, const int*, void*, size_t, int* const*, float* const*, float* const*, float* const*,
             cudaStream_t);
int coco_rank(int, const int*, const int*, const double*, int*, int*, double*, cudaStream_t);
int coco_bbox_iou(int, const int*, const int*, const long long*, const int*, const double*, const double*, const int*, double*, cudaStream_t);
int coco_oks(int, const double*, const int*, const int*, const long long*, const int*, const double*, const double*, const double*,
             const double*, double*, cudaStream_t);
int coco_masks(unsigned*, long long, int, const long long*, const int*, int, const int*, const long long*, const unsigned char*, int,
               const int*, const long long*, const unsigned*, int, int, const int*, const int*, const double*, int, const int*, long long*,
               int*, cudaStream_t);
int coco_segm_iou(int, int, const int*, const int*, const long long*, const int*, int, int, int, const int*, const long long*, const int*,
                  const unsigned*, const long long*, const int*, const int*, double*, cudaStream_t);
int coco_match(int, int, const double*, int, const double*, int, const int*, const int*, const long long*, const int*, const int*,
               const double*, const double*, const int*, const double*, int, unsigned*, int*, cudaStream_t);
int coco_accumulate(int, int, int, int, int, const int*, const int*, const int*, const int*, const int*, const double*, const unsigned*, int,
                    int, const int*, const double*, void*, size_t, double*, double*, double*, cudaStream_t);
int voc_match(int, int, int, double, const int*, const double*, const unsigned char*, const int*, const double*, int*, unsigned char*,
              cudaStream_t);
size_t box_proposal_match_workspace_bytes(int, int, int, int);
int box_proposal_match(int, int, int, int, int, int, const float*, const int*, const float*, const double*, const int*, const int*,
                       const double*, const double*, void*, size_t, float*, unsigned char*, unsigned char*, long long*, cudaStream_t);
int mask_targets(const float*, const int*, const int*, int, int, const int*, int, const int*, int, const int*, const float*, int, int,
                 float*, int*, cudaStream_t);
int keypoint_candidates(const float*, const float*, const int*, int, const int*, const int*, const int*, const int*, const int*, int, float,
                        int*, int*, cudaStream_t);
int keypoint_targets(const float*, const int*, int, const int*, const int*, const int*, const int*, const int*, int, int, const int*,
                     const int*, const int*, const int*, const float*, const float*, float*, int*, float*, cudaStream_t);
int image_blob(const unsigned char*, const b200_image_blob_desc*, int, const float*, int, int, float*, cudaStream_t);

// B200_ROI_ALIGN_PATH=generic|tiled|stream|auto (default auto) -- test/benchmark override of the forward dispatch
//   0 auto: streaming-strip path -> quad-strip path -> tiled path -> generic, each when it applies.  On H100 the streaming
//     path is at least as fast as the quad strips at every benchmarked shape (BASELINE cfg2 and FPN P2 / P4 box and mask
//     heads, DESIGN.md 4.1) and bit-exact wherever a bin's samples fit the strip, so it is tried first.
//   1 generic only; 2 tiled (-> generic); 3 stream (-> generic); 4 quad strip (-> generic)
static int forward_path_mode() {
    const int e = option_get(kOptFwdPath);
    if (e == 'g') return 1;
    if (e == 't') return 2;
    if (e == 's') return 3;
    if (e == 'q') return 4;
    return 0;
}

// The pyramid call (b200_roi_align_forward_fpn) runs the quad strips: in auto mode and under B200_ROI_ALIGN_PATH=quad.
static bool fpn_fused(int mode) { return mode == 0 || mode == 4; }

static size_t forward_workspace_bytes(int mode, int N, int R, int H, int W, int PH, int PW, int sr) {
    if (mode == 1) return 0;
    const size_t a = (mode == 3 || mode == 0) ? roi_align_stream_workspace_bytes(N, R, H, W, PH, PW, sr) : 0;
    const size_t b = (mode == 2 || mode == 0) ? roi_align_tiled_workspace_bytes(N, R, H, W, PH, PW, sr) : 0;
    const size_t c = (mode == 4 || mode == 0) ? roi_align_strip_workspace_bytes(N, R, H, W, PH, PW, sr) : 0;
    const size_t ab = a > b ? a : b;
    return ab > c ? ab : c;
}

static bool tiled_pays_off(int R, int C, int H, int W, int PH, int PW) {
    // the fast paths stream the whole map and pay a prepass; they win once the gather volume dwarfs both (BASELINE cfg1,
    // 0.4 M outputs, on an H100: generic 20 us, quad strips 28 us, stream 40 us).  The 1.5 M threshold itself has not been
    // re-measured on H100.
    const long long outputs = (long long)R * C * PH * PW;
    return outputs >= 1500000LL && (long long)H * W >= 1024;
}
int nms(const float*, int, int, float, int*, int*, void*, size_t, cudaStream_t);
size_t nms_batched_workspace_bytes(const int*, int);
int soft_nms_batched(float*, const int*, int, float, float, float, int, int*, int*, cudaStream_t);
int box_voting_batched(const float*, const int*, const float*, const int*, int, float, int, float, float*, cudaStream_t);
int nms_batched(const float*, const int*, int, int, float, bool, int*, int*, void*, size_t, cudaStream_t);
size_t roi_align_bwd_nhwc_workspace_bytes(int, int, int, int);
int roi_align_backward_nhwc(const float*, float, int, int, int, int, int, int, int, int, const float*, float*, const int*, void*, size_t, cudaStream_t);

size_t roi_align_bwd_rows_workspace_bytes(int, int, int, int, int, int, int, int);
int roi_align_backward_rows(const float*, float, int, int, int, int, int, int, int, int, const float*, float*, const int*, void*, size_t, cudaStream_t);

// B200_ROI_ALIGN_BWD_PATH=generic|nhwc|rows|auto
static int backward_path_mode() {
    const int e = option_get(kOptBwdPath);
    if (e == 'g') return 1;
    if (e == 'n') return 2;
    if (e == 'r') return 3;
    return 0;
}

static bool nhwc_pays_off(int N, int R, int C, int H, int W, int PH, int PW, int sr) {
    // fixed cost: zero + transpose the whole map; gain: 4x fewer L2 reduction ops
    if (sr < 1 || (C & 3)) return false;
    const long long taps = (long long)R * C * PH * PW * sr * sr * 4;
    return taps >= 2LL * N * C * H * W;
}

// 0: generic (scalar atomics), 2: NHWC vector reductions, 3: row-stationary gather
static int backward_path_choice(int N, int R, int C, int H, int W, int PH, int PW, int sr) {
    const int mode = backward_path_mode();
    if (mode == 1 || R <= 0) return 0;
    const bool pays = nhwc_pays_off(N, R, C, H, W, PH, PW, sr);
    bool rows_ok = roi_align_bwd_rows_workspace_bytes(N, R, C, H, W, PH, PW, sr) > 0;
    if (rows_ok && mode != 3) {
        // The gather path's parallelism is (image rows) x (32-cell tiles) x (128-channel blocks) warp items, each walking
        // every unit of its row: few rows with many RoIs (FPN P4 / P5 with a thousand boxes) leave most of the resident
        // warps (12 per SM) idle behind a few very long items.  These thresholds have not been re-measured on H100.
        // 14 x 14 bins (mask head) stay on this path: at FPN P2, 2 x 256 x 200 x 336 with 256 RoIs, it takes 238 us on an
        // H100 against 603 us for the vector-reduction path and 1169 us for the scalar-atomic kernel.
        const long long items = (long long)N * H * ((W + 31) / 32) * ((C + 127) / 128);
        const long long units_per_row = 2LL * R * PH * (sr > 0 ? sr : 1) / ((long long)N * H);
        if (items < 1200 || units_per_row > 160) rows_ok = false;
    }
    if (mode == 3) return rows_ok ? 3 : 0;
    if (mode == 2) return 2;
    if (rows_ok && pays) return 3;
    return pays ? 2 : 0;
}

static inline bool bad_dims(int N, int R, int H, int W, int C, int PH, int PW) {
    return N < 0 || R < 0 || H <= 0 || W <= 0 || C < 0 || PH <= 0 || PW <= 0;
}
}  // namespace b200

using namespace b200;

extern "C" {

int b200_roi_ops_abi_version(void) { return 3; }

const char* b200_roi_ops_strerror(int status) {
    if (status == B200_ROI_OK) return "success";
    if (status == B200_ROI_EINVAL) return "b200_roi_ops: invalid argument (null pointer, negative or zero dimension)";
    if (status == B200_ROI_EWORKSPACE) return "b200_roi_ops: workspace missing or smaller than b200_nms_workspace_bytes()";
    if (status > 0) return cudaGetErrorString((cudaError_t)status);
    return "b200_roi_ops: unknown status";
}

unsigned long long b200_roi_ops_launch_count(void) { return g_launch_count; }

int b200_roi_ops_set_option(const char* name, const char* value) { return option_set(name, value); }

void b200_roi_ops_debug_timing_buffer(void* device_u64x16) {
    nms_set_timing_buffer((unsigned long long*)device_u64x16);
    roi_align_stream_set_debug_buffer((unsigned long long*)device_u64x16);      // watchdog records of the streaming-strip path
    roi_align_strip_set_debug_buffer((unsigned long long*)device_u64x16);       // watchdog records of the quad-strip path
}

size_t b200_roi_align_workspace_bytes(int batch_size, int num_rois, int height, int width, int aligned_height,
                                      int aligned_width, int sampling_ratio) {
    if (batch_size <= 0 || num_rois <= 0 || height <= 0 || width <= 0 || aligned_height <= 0 || aligned_width <= 0) return 0;
    return forward_workspace_bytes(forward_path_mode(), batch_size, num_rois, height, width, aligned_height, aligned_width, sampling_ratio);
}

int b200_roi_align_forward_ws(const float* bottom_data, float spatial_scale, int batch_size, int num_rois, int height,
                              int width, int channels, int aligned_height, int aligned_width, int sampling_ratio,
                              const float* bottom_rois, float* top_data, void* workspace, size_t workspace_bytes,
                              b200_stream_t stream) {
    return b200_roi_align_forward_indexed(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels,
                                          aligned_height, aligned_width, sampling_ratio, bottom_rois, nullptr, top_data,
                                          workspace, workspace_bytes, stream);
}

int b200_roi_align_forward_indexed(const float* bottom_data, float spatial_scale, int batch_size, int num_rois, int height,
                                   int width, int channels, int aligned_height, int aligned_width, int sampling_ratio,
                                   const float* bottom_rois, const int* top_rows, float* top_data, void* workspace,
                                   size_t workspace_bytes, b200_stream_t stream) {
    if (bad_dims(batch_size, num_rois, height, width, channels, aligned_height, aligned_width)) return B200_ROI_EINVAL;
    if (num_rois > 0 && channels > 0 && (!bottom_data || !bottom_rois || !top_data)) return B200_ROI_EINVAL;
    const int mode = forward_path_mode();
    const bool pays = tiled_pays_off(num_rois, channels, height, width, aligned_height, aligned_width);
    if (workspace != nullptr && (mode == 3 || (mode == 0 && pays))) {
        const int rc = roi_align_forward_stream(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels,
                                                aligned_height, aligned_width, sampling_ratio, bottom_rois, top_data, top_rows,
                                                workspace, workspace_bytes, (cudaStream_t)stream);
        if (rc != kPathDeclined) return rc;
    }
    if (workspace != nullptr && (mode == 4 || (mode == 0 && pays))) {
        const int rc = roi_align_forward_strip(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels,
                                               aligned_height, aligned_width, sampling_ratio, bottom_rois, top_data, top_rows,
                                               workspace, workspace_bytes, (cudaStream_t)stream);
        if (rc != kPathDeclined) return rc;
    }
    if (workspace != nullptr && (mode == 2 || (mode == 0 && pays))) {
        const int rc = roi_align_forward_tiled(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels,
                                               aligned_height, aligned_width, sampling_ratio, bottom_rois, top_data, top_rows,
                                               workspace, workspace_bytes, (cudaStream_t)stream);
        if (rc != kPathDeclined) return rc;
    }
    return roi_align_forward_generic(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels,
                                     aligned_height, aligned_width, sampling_ratio, bottom_rois, top_data, top_rows,
                                     (cudaStream_t)stream);
}

int b200_roi_align_forward(const float* bottom_data, float spatial_scale, int batch_size, int num_rois, int height,
                           int width, int channels, int aligned_height, int aligned_width, int sampling_ratio,
                           const float* bottom_rois, float* top_data, b200_stream_t stream) {
    if (bad_dims(batch_size, num_rois, height, width, channels, aligned_height, aligned_width)) return B200_ROI_EINVAL;
    if (num_rois > 0 && channels > 0 && (!bottom_data || !bottom_rois || !top_data)) return B200_ROI_EINVAL;
    const int mode = forward_path_mode();
    const size_t wsb = (num_rois > 0) ? forward_workspace_bytes(mode, batch_size, num_rois, height, width, aligned_height, aligned_width,
                                                                sampling_ratio) : 0;
    if (wsb > 0 && (mode >= 2 || tiled_pays_off(num_rois, channels, height, width, aligned_height, aligned_width))) {
        void* ws = nullptr;
        if (cudaMallocAsync(&ws, wsb, (cudaStream_t)stream) == cudaSuccess) {
            const int rc = b200_roi_align_forward_ws(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels,
                                                     aligned_height, aligned_width, sampling_ratio, bottom_rois, top_data, ws,
                                                     wsb, stream);
            cudaFreeAsync(ws, (cudaStream_t)stream);
            return rc;
        }
        (void)cudaGetLastError();
    }
    return roi_align_forward_generic(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels,
                                     aligned_height, aligned_width, sampling_ratio, bottom_rois, top_data, nullptr,
                                     (cudaStream_t)stream);
}

size_t b200_roi_align_backward_workspace_bytes(int batch_size, int num_rois, int channels, int height, int width,
                                               int aligned_height, int aligned_width, int sampling_ratio) {
    if (batch_size <= 0 || num_rois <= 0 || channels <= 0 || height <= 0 || width <= 0 || aligned_height <= 0 || aligned_width <= 0) return 0;
    const int path = backward_path_choice(batch_size, num_rois, channels, height, width, aligned_height, aligned_width, sampling_ratio);
    if (path == 3) return roi_align_bwd_rows_workspace_bytes(batch_size, num_rois, channels, height, width, aligned_height, aligned_width, sampling_ratio);
    if (path == 2) return roi_align_bwd_nhwc_workspace_bytes(batch_size, channels, height, width);
    return 0;
}

int b200_roi_align_backward_ws(const float* top_diff, float spatial_scale, int batch_size, int num_rois, int height,
                               int width, int channels, int aligned_height, int aligned_width, int sampling_ratio,
                               const float* bottom_rois, float* bottom_diff, void* workspace, size_t workspace_bytes,
                               b200_stream_t stream) {
    return b200_roi_align_backward_indexed(top_diff, nullptr, spatial_scale, batch_size, num_rois, height, width, channels,
                                           aligned_height, aligned_width, sampling_ratio, bottom_rois, bottom_diff, workspace,
                                           workspace_bytes, stream);
}

int b200_roi_align_backward_indexed(const float* top_diff, const int* top_rows, float spatial_scale, int batch_size,
                                    int num_rois, int height, int width, int channels, int aligned_height, int aligned_width,
                                    int sampling_ratio, const float* bottom_rois, float* bottom_diff, void* workspace,
                                    size_t workspace_bytes, b200_stream_t stream) {
    if (bad_dims(batch_size, num_rois, height, width, channels, aligned_height, aligned_width)) return B200_ROI_EINVAL;
    if ((size_t)batch_size * channels == 0) return B200_ROI_OK;
    if (!bottom_diff || (num_rois > 0 && (!top_diff || !bottom_rois))) return B200_ROI_EINVAL;
    int path = (workspace != nullptr) ? backward_path_choice(batch_size, num_rois, channels, height, width, aligned_height, aligned_width, sampling_ratio) : 0;
    if (path == 3) {
        const int rc = roi_align_backward_rows(top_diff, spatial_scale, batch_size, num_rois, height, width, channels,
                                               aligned_height, aligned_width, sampling_ratio, bottom_rois, bottom_diff,
                                               top_rows, workspace, workspace_bytes, (cudaStream_t)stream);
        if (rc != kPathDeclined) return rc;
        path = 2;                                   // workspace too small for the gather path: try the NHWC one
    }
    if (path == 2) {
        const int rc = roi_align_backward_nhwc(top_diff, spatial_scale, batch_size, num_rois, height, width, channels,
                                               aligned_height, aligned_width, sampling_ratio, bottom_rois, bottom_diff,
                                               top_rows, workspace, workspace_bytes, (cudaStream_t)stream);
        if (rc != kPathDeclined) return rc;
    }
    return roi_align_backward_generic(top_diff, spatial_scale, batch_size, num_rois, height, width, channels,
                                      aligned_height, aligned_width, sampling_ratio, bottom_rois, bottom_diff, top_rows,
                                      (cudaStream_t)stream);
}

int b200_roi_align_backward(const float* top_diff, float spatial_scale, int batch_size, int num_rois, int height,
                            int width, int channels, int aligned_height, int aligned_width, int sampling_ratio,
                            const float* bottom_rois, float* bottom_diff, b200_stream_t stream) {
    if (bad_dims(batch_size, num_rois, height, width, channels, aligned_height, aligned_width)) return B200_ROI_EINVAL;
    if ((size_t)batch_size * channels == 0) return B200_ROI_OK;
    if (!bottom_diff || (num_rois > 0 && (!top_diff || !bottom_rois))) return B200_ROI_EINVAL;
    const size_t wsb = b200_roi_align_backward_workspace_bytes(batch_size, num_rois, channels, height, width, aligned_height,
                                                               aligned_width, sampling_ratio);
    if (wsb > 0) {
        void* ws = nullptr;
        if (cudaMallocAsync(&ws, wsb, (cudaStream_t)stream) == cudaSuccess) {
            const int rc = b200_roi_align_backward_ws(top_diff, spatial_scale, batch_size, num_rois, height, width, channels,
                                                      aligned_height, aligned_width, sampling_ratio, bottom_rois, bottom_diff,
                                                      ws, wsb, stream);
            cudaFreeAsync(ws, (cudaStream_t)stream);
            return rc;
        }
        (void)cudaGetLastError();
    }
    return roi_align_backward_generic(top_diff, spatial_scale, batch_size, num_rois, height, width, channels,
                                      aligned_height, aligned_width, sampling_ratio, bottom_rois, bottom_diff, nullptr,
                                      (cudaStream_t)stream);
}

int b200_proposal_decode(const float* bbox_deltas, const float* anchors, const long long* order, const float* scores,
                         int num_candidates, int num_anchors, int height, int width, float feat_stride, float im_height,
                         float im_width, float min_size, float* dets_out, int* valid_out, b200_stream_t stream) {
    if (num_candidates < 0 || num_anchors <= 0 || height <= 0 || width <= 0) return B200_ROI_EINVAL;
    if (num_candidates > 0 && (!bbox_deltas || !anchors || !order || !scores || !dets_out || !valid_out)) return B200_ROI_EINVAL;
    return proposal_decode(bbox_deltas, anchors, order, scores, num_candidates, num_anchors, height, width, feat_stride,
                           im_height, im_width, min_size, dets_out, valid_out, (cudaStream_t)stream);
}

int b200_roi_align_legacy_forward(const float* bottom_data, float spatial_scale, int batch_size, int num_rois,
                                  int height, int width, int channels, int aligned_height, int aligned_width,
                                  const float* bottom_rois, float* top_data, b200_stream_t stream) {
    if (bad_dims(batch_size, num_rois, height, width, channels, aligned_height, aligned_width)) return B200_ROI_EINVAL;
    if (num_rois > 0 && channels > 0 && (!bottom_data || !bottom_rois || !top_data)) return B200_ROI_EINVAL;
    return roi_align_legacy_forward(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels,
                                    aligned_height, aligned_width, bottom_rois, top_data, (cudaStream_t)stream);
}

int b200_roi_align_legacy_backward(const float* top_diff, float spatial_scale, int batch_size, int num_rois,
                                   int height, int width, int channels, int aligned_height, int aligned_width,
                                   const float* bottom_rois, float* bottom_diff, b200_stream_t stream) {
    if (bad_dims(batch_size, num_rois, height, width, channels, aligned_height, aligned_width)) return B200_ROI_EINVAL;
    if ((size_t)batch_size * channels == 0) return B200_ROI_OK;
    if (!bottom_diff || (num_rois > 0 && (!top_diff || !bottom_rois))) return B200_ROI_EINVAL;
    return roi_align_legacy_backward(top_diff, spatial_scale, batch_size, num_rois, height, width, channels,
                                     aligned_height, aligned_width, bottom_rois, bottom_diff, (cudaStream_t)stream);
}

int b200_roi_pool_forward(const float* bottom_data, float spatial_scale, int batch_size, int num_rois, int height,
                          int width, int channels, int pooled_height, int pooled_width, const float* bottom_rois,
                          float* top_data, int* argmax_data, b200_stream_t stream) {
    if (bad_dims(batch_size, num_rois, height, width, channels, pooled_height, pooled_width)) return B200_ROI_EINVAL;
    if (num_rois > 0 && channels > 0 && (!bottom_data || !bottom_rois || !top_data)) return B200_ROI_EINVAL;
    return roi_pool_forward(bottom_data, spatial_scale, batch_size, num_rois, height, width, channels, pooled_height,
                            pooled_width, bottom_rois, top_data, argmax_data, (cudaStream_t)stream);
}

int b200_roi_pool_backward(const float* top_diff, float spatial_scale, int batch_size, int num_rois, int height,
                           int width, int channels, int pooled_height, int pooled_width, const float* bottom_rois,
                           float* bottom_diff, const int* argmax_data, b200_stream_t stream) {
    if (bad_dims(batch_size, num_rois, height, width, channels, pooled_height, pooled_width)) return B200_ROI_EINVAL;
    if ((size_t)batch_size * channels == 0) return B200_ROI_OK;
    if (!bottom_diff || (num_rois > 0 && (!top_diff || !bottom_rois || !argmax_data))) return B200_ROI_EINVAL;
    return roi_pool_backward(top_diff, spatial_scale, batch_size, num_rois, height, width, channels, pooled_height,
                             pooled_width, bottom_rois, bottom_diff, argmax_data, (cudaStream_t)stream);
}

int b200_roi_crop_forward(const float* image, const float* grids, int batch_size, int channels, int height, int width,
                          int num_rois, int out_height, int out_width, float* output, b200_stream_t stream) {
    if (batch_size < 0 || channels < 0 || height <= 0 || width <= 0 || num_rois < 0 || out_height < 0 || out_width < 0)
        return B200_ROI_EINVAL;
    if ((size_t)num_rois * out_height * out_width * channels > 0 && (!image || !grids || !output)) return B200_ROI_EINVAL;
    return roi_crop_forward(image, grids, batch_size, channels, height, width, num_rois, out_height, out_width, output,
                            (cudaStream_t)stream);
}

int b200_roi_crop_backward(const float* grad_output, const float* grids, int batch_size, int channels, int height,
                           int width, int num_rois, int out_height, int out_width, float* grad_image,
                           float* grad_grids, b200_stream_t stream) {
    if (batch_size < 0 || channels < 0 || height <= 0 || width <= 0 || num_rois < 0 || out_height < 0 || out_width < 0)
        return B200_ROI_EINVAL;
    if ((size_t)batch_size * channels == 0) return B200_ROI_OK;
    if (!grad_image) return B200_ROI_EINVAL;
    if ((size_t)num_rois * out_height * out_width > 0 && (!grad_output || !grids)) return B200_ROI_EINVAL;
    return roi_crop_backward(grad_output, grids, batch_size, channels, height, width, num_rois, out_height, out_width,
                             grad_image, grad_grids, nullptr, 0, (cudaStream_t)stream);
}

size_t b200_roi_crop_backward_workspace_bytes(int batch_size, int channels, int height, int width, int num_rois, int out_height,
                                              int out_width) {
    if (batch_size <= 0 || channels <= 0 || height <= 0 || width <= 0 || num_rois <= 0 || out_height <= 0 || out_width <= 0) return 0;
    return roi_crop_backward_workspace_bytes(batch_size, channels, height, width, num_rois, out_height, out_width);
}

int b200_roi_crop_backward_ws(const float* grad_output, const float* grids, int batch_size, int channels, int height, int width,
                              int num_rois, int out_height, int out_width, float* grad_image, float* grad_grids, void* workspace,
                              size_t workspace_bytes, b200_stream_t stream) {
    if (batch_size < 0 || channels < 0 || height <= 0 || width <= 0 || num_rois < 0 || out_height < 0 || out_width < 0)
        return B200_ROI_EINVAL;
    if ((size_t)batch_size * channels == 0) return B200_ROI_OK;
    if (!grad_image) return B200_ROI_EINVAL;
    if ((size_t)num_rois * out_height * out_width > 0 && (!grad_output || !grids)) return B200_ROI_EINVAL;
    return roi_crop_backward(grad_output, grids, batch_size, channels, height, width, num_rois, out_height, out_width,
                             grad_image, grad_grids, workspace, workspace_bytes, (cudaStream_t)stream);
}

size_t b200_nms_workspace_bytes(int boxes_num) { return nms_workspace_bytes(boxes_num); }

int b200_nms(const float* boxes_dev, int boxes_num, int boxes_dim, float nms_overlap_thresh, int* keep_out_dev,
             int* num_out_dev, void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    if (!num_out_dev || (boxes_num > 0 && (!boxes_dev || !keep_out_dev))) return B200_ROI_EINVAL;
    return nms(boxes_dev, boxes_num, boxes_dim, nms_overlap_thresh, keep_out_dev, num_out_dev, workspace,
               workspace_bytes, (cudaStream_t)stream);
}

size_t b200_roi_align_fpn_workspace_bytes(int num_levels, const int* heights_host, const int* widths_host, int batch_size, int num_rois,
                                          int aligned_height, int aligned_width, int sampling_ratio) {
    if (num_levels < 1 || !heights_host || !widths_host || batch_size <= 0 || num_rois <= 0 || !fpn_fused(forward_path_mode())) return 0;
    return roi_align_strip_fpn_workspace_bytes(num_levels, heights_host, widths_host, batch_size, num_rois, aligned_height, aligned_width,
                                               sampling_ratio);
}

int b200_roi_align_forward_fpn(int num_levels, const float* const* bottom_data_host, const int* heights_host, const int* widths_host,
                               const float* spatial_scales_host, const int* level_roi_begin_host, int batch_size, int num_rois,
                               int channels, int aligned_height, int aligned_width, int sampling_ratio, const float* bottom_rois,
                               const int* top_rows, float* top_data, void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    if (num_levels < 1 || num_levels > 6 || !bottom_data_host || !heights_host || !widths_host || !spatial_scales_host || !level_roi_begin_host)
        return B200_ROI_EINVAL;
    if (batch_size <= 0 || num_rois <= 0 || channels <= 0 || aligned_height <= 0 || aligned_width <= 0 || !bottom_rois || !top_data)
        return B200_ROI_EINVAL;
    if (level_roi_begin_host[0] != 0 || level_roi_begin_host[num_levels] != num_rois) return B200_ROI_EINVAL;
    for (int l = 0; l < num_levels; ++l)
        if (!bottom_data_host[l] || level_roi_begin_host[l + 1] < level_roi_begin_host[l]) return B200_ROI_EINVAL;
    int rc = kPathDeclined;
    if (fpn_fused(forward_path_mode())) {
        // Levels that TMA can stage (W % 4 == 0, 16-byte aligned base) and levels that need the cp.async producers (FPN P5 of an
        // 800 x 1333 image: W = 42) go to separate launch sequences: runs of consecutive levels of the same kind, each over its
        // own contiguous range of the level-major RoIs.  The workspace is reused (stream order).
        const int bins = aligned_height * aligned_width;
        int l0 = 0;
        rc = B200_ROI_OK;
        while (l0 < num_levels && rc == B200_ROI_OK) {
            auto tma_ok = [&](int l) { return (widths_host[l] & 3) == 0 && ((uintptr_t)bottom_data_host[l] & 15u) == 0; };
            int l1 = l0 + 1;
            while (l1 < num_levels && tma_ok(l1) == tma_ok(l0)) ++l1;
            const int r0 = level_roi_begin_host[l0], r1 = level_roi_begin_host[l1];
            if (r1 > r0) {
                int begin[8];
                for (int l = l0; l <= l1; ++l) begin[l - l0] = level_roi_begin_host[l] - r0;
                rc = roi_align_forward_strip_fpn(l1 - l0, bottom_data_host + l0, heights_host + l0, widths_host + l0, spatial_scales_host + l0,
                                                 begin, batch_size, r1 - r0, channels, aligned_height, aligned_width, sampling_ratio,
                                                 bottom_rois + (size_t)5 * r0, top_rows ? top_data : top_data + (size_t)r0 * channels * bins,
                                                 top_rows ? top_rows + r0 : nullptr, workspace, workspace_bytes, (cudaStream_t)stream);
            }
            l0 = l1;
        }
        if (rc != B200_ROI_OK && rc != kPathDeclined) return rc;
    }
    return rc == kPathDeclined ? B200_ROI_EWORKSPACE : rc;
}

size_t b200_nms_batched_workspace_bytes(const int* counts_host, int num_problems) {
    if (!counts_host) return 0;
    return nms_batched_workspace_bytes(counts_host, num_problems);
}

static int nms_batched_entry(const float* boxes_dev, const int* counts_host, int num_problems, int boxes_dim, float nms_overlap_thresh,
                             bool cython, int* keep_out_dev, int* num_out_dev, void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    if (!counts_host || num_problems < 1 || !num_out_dev) return B200_ROI_EINVAL;
    long long total = 0;
    for (int p = 0; p < num_problems && p < 64; ++p) total += counts_host[p] > 0 ? counts_host[p] : 0;
    if (total > 0 && (!boxes_dev || !keep_out_dev)) return B200_ROI_EINVAL;
    const int rc = nms_batched(boxes_dev, counts_host, num_problems, boxes_dim, nms_overlap_thresh, cython, keep_out_dev, num_out_dev,
                               workspace, workspace_bytes, (cudaStream_t)stream);
    return rc == kPathDeclined ? B200_ROI_EINVAL : rc;
}

int b200_nms_batched(const float* boxes_dev, const int* counts_host, int num_problems, int boxes_dim, float nms_overlap_thresh,
                     int* keep_out_dev, int* num_out_dev, void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    return nms_batched_entry(boxes_dev, counts_host, num_problems, boxes_dim, nms_overlap_thresh, false, keep_out_dev, num_out_dev, workspace,
                             workspace_bytes, stream);
}

int b200_nms_batched_cython(const float* boxes_dev, const int* counts_host, int num_problems, int boxes_dim, float nms_overlap_thresh,
                            int* keep_out_dev, int* num_out_dev, void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    return nms_batched_entry(boxes_dev, counts_host, num_problems, boxes_dim, nms_overlap_thresh, true, keep_out_dev, num_out_dev, workspace,
                             workspace_bytes, stream);
}

int b200_soft_nms_batched(float* dets_dev, const int* counts_host, int num_problems, float sigma, float overlap_thresh,
                          float score_thresh, int method, int* inds_out_dev, int* num_out_dev, b200_stream_t stream) {
    if (!counts_host || num_problems < 1 || !num_out_dev) return B200_ROI_EINVAL;
    long long total = 0;
    for (int p = 0; p < num_problems && p < 128; ++p) total += counts_host[p] > 0 ? counts_host[p] : 0;
    if (total > 0 && (!dets_dev || !inds_out_dev)) return B200_ROI_EINVAL;
    return soft_nms_batched(dets_dev, counts_host, num_problems, sigma, overlap_thresh, score_thresh, method, inds_out_dev, num_out_dev,
                            (cudaStream_t)stream);
}

int b200_box_voting_batched(const float* top_dets_dev, const int* top_counts_host, const float* all_dets_dev, const int* all_counts_host,
                            int num_problems, float thresh, int scoring_method, float beta, float* out_dev, b200_stream_t stream) {
    if (!top_counts_host || !all_counts_host || num_problems < 1) return B200_ROI_EINVAL;
    long long total = 0;
    for (int p = 0; p < num_problems && p < 128; ++p) total += top_counts_host[p] > 0 ? top_counts_host[p] : 0;
    if (total > 0 && (!top_dets_dev || !all_dets_dev || !out_dev)) return B200_ROI_EINVAL;
    if (scoring_method < 0 || scoring_method > 5) return B200_ROI_EINVAL;
    return box_voting_batched(top_dets_dev, top_counts_host, all_dets_dev, all_counts_host, num_problems, thresh, scoring_method, beta, out_dev,
                              (cudaStream_t)stream);
}

size_t b200_topk_batched_workspace_bytes(int num_problems) { return topk_batched_workspace_bytes(num_problems); }

int b200_topk_batched(const float* const* scores_dev_ptrs_host, const int* num_anchors_host, const int* num_cells_host, const int* k_host,
                      int num_problems, long long* order_out_dev, float* scores_out_dev, void* workspace, size_t workspace_bytes,
                      b200_stream_t stream) {
    if (num_problems < 1 || !scores_dev_ptrs_host || !num_anchors_host || !num_cells_host || !k_host) return B200_ROI_EINVAL;
    long long total = 0;
    for (int p = 0; p < num_problems && p < 64; ++p) {
        if (!scores_dev_ptrs_host[p] || k_host[p] < 0) return B200_ROI_EINVAL;
        total += k_host[p];
    }
    if (total > 0 && (!order_out_dev || !scores_out_dev)) return B200_ROI_EINVAL;
    const int rc = topk_batched(scores_dev_ptrs_host, num_anchors_host, num_cells_host, k_host, num_problems, order_out_dev, scores_out_dev,
                                workspace, workspace_bytes, (cudaStream_t)stream);
    return rc == kPathDeclined ? B200_ROI_EWORKSPACE : rc;
}

int b200_bbox_overlaps(const float* boxes_dev, int num_boxes, const float* query_boxes_dev, int num_query, float* overlaps_out_dev,
                       b200_stream_t stream) {
    if (num_boxes < 0 || num_query < 0) return B200_ROI_EINVAL;
    if ((long long)num_boxes * num_query > 0 && (!boxes_dev || !query_boxes_dev || !overlaps_out_dev)) return B200_ROI_EINVAL;
    return bbox_overlaps(boxes_dev, num_boxes, query_boxes_dev, num_query, overlaps_out_dev, (cudaStream_t)stream);
}

int b200_roi_assign(const float* boxes_dev, int num_boxes, const float* gt_boxes_dev, const int* gt_classes_dev, int num_gt,
                    float* max_overlaps_out_dev, int* argmax_out_dev, int* max_classes_out_dev, b200_stream_t stream) {
    if (num_boxes < 0 || num_gt < 0) return B200_ROI_EINVAL;
    if (num_boxes > 0 && (!boxes_dev || !max_overlaps_out_dev || !argmax_out_dev || !max_classes_out_dev)) return B200_ROI_EINVAL;
    if (num_boxes > 0 && num_gt > 0 && (!gt_boxes_dev || !gt_classes_dev)) return B200_ROI_EINVAL;
    return roi_assign(boxes_dev, num_boxes, gt_boxes_dev, gt_classes_dev, num_gt, max_overlaps_out_dev, argmax_out_dev, max_classes_out_dev,
                      (cudaStream_t)stream);
}

int b200_roi_select(const float* max_overlaps_dev, int num_boxes, float fg_thresh, float bg_thresh_hi, float bg_thresh_lo,
                    int* fg_inds_out_dev, int* bg_inds_out_dev, int* counts_out_dev, b200_stream_t stream) {
    if (num_boxes < 0 || !counts_out_dev) return B200_ROI_EINVAL;
    if (num_boxes > 0 && (!max_overlaps_dev || !fg_inds_out_dev || !bg_inds_out_dev)) return B200_ROI_EINVAL;
    return roi_select(max_overlaps_dev, num_boxes, fg_thresh, bg_thresh_hi, bg_thresh_lo, fg_inds_out_dev, bg_inds_out_dev, counts_out_dev,
                      (cudaStream_t)stream);
}

int b200_fast_rcnn_targets(const float* boxes_dev, const float* gt_boxes_dev, const int* argmax_dev, const int* max_classes_dev,
                           const int* keep_inds_dev, int num_keep, int num_fg, const float* bbox_reg_weights_host, int num_reg_classes,
                           int cls_agnostic, float im_scale, float batch_idx, int* labels_out_dev, float* rois_out_dev,
                           float* bbox_targets_out_dev, float* inside_weights_out_dev, float* outside_weights_out_dev,
                           b200_stream_t stream) {
    if (num_keep < 0 || num_fg < 0 || num_fg > num_keep || num_reg_classes < 1 || !bbox_reg_weights_host) return B200_ROI_EINVAL;
    if (num_keep > 0 && (!boxes_dev || !argmax_dev || !max_classes_dev || !keep_inds_dev || !labels_out_dev || !rois_out_dev ||
                         !bbox_targets_out_dev || !inside_weights_out_dev || !outside_weights_out_dev))
        return B200_ROI_EINVAL;
    return fast_rcnn_targets(boxes_dev, gt_boxes_dev, argmax_dev, max_classes_dev, keep_inds_dev, num_keep, num_fg, bbox_reg_weights_host,
                             num_reg_classes, cls_agnostic, im_scale, batch_idx, labels_out_dev, rois_out_dev, bbox_targets_out_dev,
                             inside_weights_out_dev, outside_weights_out_dev, (cudaStream_t)stream);
}

size_t b200_segm_workspace_bytes(int num_dets) { return segm_workspace_bytes(num_dets); }

int b200_segm_rle_sizes(const float* masks_dev, const int* mask_class_dev, const float* boxes_dev, int num_dets, int num_channels,
                        int resolution, int im_h, int im_w, float thresh, int* sizes_out_dev, void* workspace, size_t workspace_bytes,
                        b200_stream_t stream) {
    if (!segm_args_ok(num_dets, num_channels, resolution, im_h, im_w)) return B200_ROI_EINVAL;
    if (num_dets == 0) return B200_ROI_OK;
    if (!masks_dev || !mask_class_dev || !boxes_dev || !sizes_out_dev) return B200_ROI_EINVAL;
    if (!workspace || workspace_bytes < segm_workspace_bytes(num_dets)) return B200_ROI_EWORKSPACE;
    return segm_rle_sizes(masks_dev, mask_class_dev, boxes_dev, num_dets, num_channels, resolution, im_h, im_w, thresh, sizes_out_dev,
                          workspace, (cudaStream_t)stream);
}

int b200_segm_rle_emit(const float* masks_dev, const int* mask_class_dev, const float* boxes_dev, int num_dets, int num_channels,
                       int resolution, int im_h, int im_w, float thresh, const int* sizes_dev, const void* workspace,
                       size_t workspace_bytes, int* counts_out_dev, long long* count_offsets_out_dev, unsigned char* strings_out_dev,
                       long long* string_offsets_out_dev, b200_stream_t stream) {
    if (!segm_args_ok(num_dets, num_channels, resolution, im_h, im_w)) return B200_ROI_EINVAL;
    if (num_dets == 0) return B200_ROI_OK;
    if (!masks_dev || !mask_class_dev || !boxes_dev || !sizes_dev || !counts_out_dev || !count_offsets_out_dev || !strings_out_dev ||
        !string_offsets_out_dev)
        return B200_ROI_EINVAL;
    if (!workspace || workspace_bytes < segm_workspace_bytes(num_dets)) return B200_ROI_EWORKSPACE;
    return segm_rle_emit(masks_dev, mask_class_dev, boxes_dev, num_dets, num_channels, resolution, im_h, im_w, thresh, sizes_dev,
                         workspace, counts_out_dev, count_offsets_out_dev, strings_out_dev, string_offsets_out_dev, (cudaStream_t)stream);
}

int b200_paste_masks(const float* masks_dev, const int* mask_class_dev, const float* boxes_dev, int num_dets, int num_channels,
                     int resolution, int im_h, int im_w, float thresh, unsigned char* out_dev, b200_stream_t stream) {
    if (!segm_args_ok(num_dets, num_channels, resolution, im_h, im_w) || num_dets > 65535) return B200_ROI_EINVAL;
    if (num_dets == 0) return B200_ROI_OK;
    if (!masks_dev || !mask_class_dev || !boxes_dev || !out_dev) return B200_ROI_EINVAL;
    return paste_masks(masks_dev, mask_class_dev, boxes_dev, num_dets, num_channels, resolution, im_h, im_w, thresh, out_dev,
                       (cudaStream_t)stream);
}

int b200_heatmaps_to_keypoints(const float* maps_dev, const float* rois_dev, int num_rois, int num_keypoints, int heatmap_size,
                               int min_size, float* xy_preds_dev, b200_stream_t stream) {
    if (!keypoints_args_ok(num_rois, num_keypoints, heatmap_size, min_size)) return B200_ROI_EINVAL;
    if (num_rois == 0) return B200_ROI_OK;
    if (!maps_dev || !rois_dev || !xy_preds_dev) return B200_ROI_EINVAL;
    return heatmaps_to_keypoints(maps_dev, rois_dev, num_rois, num_keypoints, heatmap_size, min_size, xy_preds_dev, (cudaStream_t)stream);
}

int b200_nms_oks(const float* xy_preds_dev, const float* rois_dev, int num_rois, int num_keypoints, double thresh, int* keep_dev,
                 int* num_keep_dev, b200_stream_t stream) {
    if (!nms_oks_args_ok(num_rois, num_keypoints)) return B200_ROI_EINVAL;
    if (num_rois == 0) return B200_ROI_OK;
    if (!xy_preds_dev || !rois_dev || !keep_dev || !num_keep_dev) return B200_ROI_EINVAL;
    return nms_oks(xy_preds_dev, rois_dev, num_rois, thresh, keep_dev, num_keep_dev, (cudaStream_t)stream);
}

size_t b200_rpn_targets_workspace_bytes(int num_levels, const int* field_sizes_host, const int* num_cell_anchors_host, int num_images,
                                        int num_gt_total) {
    const int total = rpn_total_anchors(num_levels, field_sizes_host, num_cell_anchors_host);
    return total < 0 ? 0 : rpn_workspace_bytes(num_images, total, num_gt_total);
}

int b200_rpn_labels(int num_levels, const int* field_sizes_host, const int* num_cell_anchors_host, const double* strides_host,
                    const double* cell_anchors_host, int num_images, const double* im_sizes_host, const int* gt_begin_host,
                    const float* gt_boxes_dev, double straddle_thresh, float positive_overlap, float negative_overlap, int* counts_out_dev,
                    void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    return rpn_labels(num_levels, field_sizes_host, num_cell_anchors_host, strides_host, cell_anchors_host, num_images, im_sizes_host,
                      gt_begin_host, gt_boxes_dev, straddle_thresh, positive_overlap, negative_overlap, counts_out_dev, workspace,
                      workspace_bytes, (cudaStream_t)stream);
}

int b200_rpn_emit(int num_levels, const int* field_sizes_host, const int* num_cell_anchors_host, const double* strides_host,
                  const double* cell_anchors_host, int num_images, const double* im_sizes_host, const int* gt_begin_host,
                  const float* gt_boxes_dev, double straddle_thresh, const int* counts_dev, const int* fg_disable_dev,
                  const int* fg_disable_begin_host, const int* bg_enable_dev, const int* bg_enable_begin_host, void* workspace,
                  size_t workspace_bytes, int* const* labels_out_host, float* const* bbox_targets_out_host,
                  float* const* inside_weights_out_host, float* const* outside_weights_out_host, b200_stream_t stream) {
    return rpn_emit(num_levels, field_sizes_host, num_cell_anchors_host, strides_host, cell_anchors_host, num_images, im_sizes_host,
                    gt_begin_host, gt_boxes_dev, straddle_thresh, counts_dev, fg_disable_dev, fg_disable_begin_host, bg_enable_dev,
                    bg_enable_begin_host, workspace, workspace_bytes, labels_out_host, bbox_targets_out_host, inside_weights_out_host,
                    outside_weights_out_host, (cudaStream_t)stream);
}

int b200_mask_targets(const float* rois_dev, const int* roi_image_dev, const int* roi_class_dev, int num_rois, int num_images,
                      const int* obj_begin_host, int num_polys, const int* poly_begin_dev, int num_coords, const int* coord_begin_dev,
                      const float* coords_dev, int resolution, int num_classes, float* obj_boxes_out_dev, int* masks_out_dev,
                      b200_stream_t stream) {
    return mask_targets(rois_dev, roi_image_dev, roi_class_dev, num_rois, num_images, obj_begin_host, num_polys, poly_begin_dev, num_coords,
                        coord_begin_dev, coords_dev, resolution, num_classes, obj_boxes_out_dev, masks_out_dev, (cudaStream_t)stream);
}

int b200_keypoint_candidates(const float* boxes_dev, const float* max_overlaps_dev, const int* box_to_gt_dev, int num_images,
                             const int* box_begin_host, const int* gt_inds_dev, const int* gt_begin_host, const int* keypoints_dev,
                             const int* person_begin_host, int num_keypoints, float fg_thresh, int* candidates_out_dev,
                             int* counts_out_dev, b200_stream_t stream) {
    return keypoint_candidates(boxes_dev, max_overlaps_dev, box_to_gt_dev, num_images, box_begin_host, gt_inds_dev, gt_begin_host,
                               keypoints_dev, person_begin_host, num_keypoints, fg_thresh, candidates_out_dev, counts_out_dev,
                               (cudaStream_t)stream);
}

int b200_keypoint_targets(const float* boxes_dev, const int* box_to_gt_dev, int num_images, const int* box_begin_host,
                          const int* gt_inds_dev, const int* gt_begin_host, const int* keypoints_dev, const int* person_begin_host,
                          int num_keypoints, int heatmap_size, const int* candidates_dev, const int* counts_dev, const int* picks_dev,
                          const int* roi_begin_host, const float* im_scales_host, const float* batch_index_host, float* rois_out_dev,
                          int* locations_out_dev, float* weights_out_dev, b200_stream_t stream) {
    return keypoint_targets(boxes_dev, box_to_gt_dev, num_images, box_begin_host, gt_inds_dev, gt_begin_host, keypoints_dev,
                            person_begin_host, num_keypoints, heatmap_size, candidates_dev, counts_dev, picks_dev, roi_begin_host,
                            im_scales_host, batch_index_host, rois_out_dev, locations_out_dev, weights_out_dev, (cudaStream_t)stream);
}

int b200_image_blob(const unsigned char* src_dev, const b200_image_blob_desc* descs_dev, int num_images, const float* mean_table_dev,
                    int blob_h, int blob_w, float* out_dev, b200_stream_t stream) {
    return image_blob(src_dev, descs_dev, num_images, mean_table_dev, blob_h, blob_w, out_dev, (cudaStream_t)stream);
}

int b200_coco_rank(int num_pairs, const int* pair_det_begin_dev, const int* pair_entry_begin_dev, const double* det_score_dev,
                   int* entry_det_out_dev, int* entry_rank_out_dev, double* entry_score_out_dev, b200_stream_t stream) {
    return coco_rank(num_pairs, pair_det_begin_dev, pair_entry_begin_dev, det_score_dev, entry_det_out_dev, entry_rank_out_dev,
                     entry_score_out_dev, (cudaStream_t)stream);
}

int b200_coco_bbox_iou(int num_pairs, const int* pair_gt_begin_dev, const int* pair_entry_begin_dev, const long long* pair_iou_begin_dev,
                       const int* entry_det_dev, const double* det_box_dev, const double* gt_box_dev, const int* gt_flags_dev,
                       double* ious_out_dev, b200_stream_t stream) {
    return coco_bbox_iou(num_pairs, pair_gt_begin_dev, pair_entry_begin_dev, pair_iou_begin_dev, entry_det_dev, det_box_dev, gt_box_dev,
                         gt_flags_dev, ious_out_dev, (cudaStream_t)stream);
}

int b200_coco_oks(int num_pairs, const double* vars_host, const int* pair_gt_begin_dev, const int* pair_entry_begin_dev,
                  const long long* pair_iou_begin_dev, const int* entry_det_dev, const double* det_kp_dev, const double* gt_kp_dev,
                  const double* gt_box_dev, const double* gt_area_dev, double* ious_out_dev, b200_stream_t stream) {
    return coco_oks(num_pairs, vars_host, pair_gt_begin_dev, pair_entry_begin_dev, pair_iou_begin_dev, entry_det_dev, det_kp_dev, gt_kp_dev,
                    gt_box_dev, gt_area_dev, ious_out_dev, (cudaStream_t)stream);
}

int b200_coco_masks(unsigned* words_dev, long long num_words, int num_slots, const long long* slot_word_dev, const int* slot_hw_dev,
                    int num_strings, const int* str_slot_dev, const long long* str_begin_dev, const unsigned char* str_bytes_dev,
                    int num_counts, const int* cnt_slot_dev, const long long* cnt_begin_dev, const unsigned* counts_dev,
                    int num_polys, int num_vertices, const int* poly_slot_dev, const int* vtx_begin_dev, const double* xy_dev,
                    int num_masks, const int* mask_slot_begin_dev, long long* mask_area_out_dev, int* mask_range_out_dev,
                    b200_stream_t stream) {
    return coco_masks(words_dev, num_words, num_slots, slot_word_dev, slot_hw_dev, num_strings, str_slot_dev, str_begin_dev, str_bytes_dev,
                      num_counts, cnt_slot_dev, cnt_begin_dev, counts_dev, num_polys, num_vertices, poly_slot_dev, vtx_begin_dev, xy_dev,
                      num_masks, mask_slot_begin_dev, mask_area_out_dev, mask_range_out_dev, (cudaStream_t)stream);
}

int b200_coco_segm_iou(int pair_begin, int num_pairs, const int* pair_gt_begin_dev, const int* pair_entry_begin_dev,
                       const long long* pair_iou_begin_dev, const int* entry_det_dev, int det0, int gt0, int gt_mask0,
                       const int* mask_slot_begin_dev, const long long* slot_word_dev, const int* slot_hw_dev, const unsigned* words_dev,
                       const long long* mask_area_dev, const int* mask_range_dev, const int* gt_flags_dev, double* ious_out_dev,
                       b200_stream_t stream) {
    return coco_segm_iou(pair_begin, num_pairs, pair_gt_begin_dev, pair_entry_begin_dev, pair_iou_begin_dev, entry_det_dev, det0, gt0,
                         gt_mask0, mask_slot_begin_dev, slot_word_dev, slot_hw_dev, words_dev, mask_area_dev, mask_range_dev, gt_flags_dev,
                         ious_out_dev, (cudaStream_t)stream);
}

int b200_coco_match(int num_pairs, int num_thresholds, const double* iou_thrs_host, int num_areas, const double* area_rng_host, int max_gt,
                    const int* pair_gt_begin_dev, const int* pair_entry_begin_dev, const long long* pair_iou_begin_dev,
                    const int* pair_cat_dev, const int* entry_det_dev, const double* det_area_dev, const double* gt_area_dev,
                    const int* gt_flags_dev, const double* ious_dev, int num_entries, unsigned* entry_flags_dev, int* npig_dev,
                    b200_stream_t stream) {
    return coco_match(num_pairs, num_thresholds, iou_thrs_host, num_areas, area_rng_host, max_gt, pair_gt_begin_dev, pair_entry_begin_dev,
                      pair_iou_begin_dev, pair_cat_dev, entry_det_dev, det_area_dev, gt_area_dev, gt_flags_dev, ious_dev, num_entries,
                      entry_flags_dev, npig_dev, (cudaStream_t)stream);
}

int b200_coco_accumulate(int num_cats, int num_areas, int num_max_dets, int num_thresholds, int num_recall, const int* max_dets_host,
                         const int* cat_entry_begin_dev, const int* cat_pairs_dev, const int* order_dev, const int* entry_rank_dev,
                         const double* entry_score_dev, const unsigned* entry_flags_dev, int num_entries, int max_cat_entries,
                         const int* npig_dev, const double* rec_thrs_dev, void* workspace, size_t workspace_bytes, double* precision_out_dev,
                         double* recall_out_dev, double* scores_out_dev, b200_stream_t stream) {
    return coco_accumulate(num_cats, num_areas, num_max_dets, num_thresholds, num_recall, max_dets_host, cat_entry_begin_dev, cat_pairs_dev,
                           order_dev, entry_rank_dev, entry_score_dev, entry_flags_dev, num_entries, max_cat_entries, npig_dev, rec_thrs_dev, workspace,
                           workspace_bytes, precision_out_dev, recall_out_dev, scores_out_dev, (cudaStream_t)stream);
}

int b200_voc_match(int num_dets, int num_pairs, int num_gt, double ovthresh, const int* pair_gt_begin_dev, const double* gt_box_dev,
                   const unsigned char* gt_difficult_dev, const int* det_pair_dev, const double* det_box_dev, int* workspace_dev,
                   unsigned char* outcome_out_dev, b200_stream_t stream) {
    return voc_match(num_dets, num_pairs, num_gt, ovthresh, pair_gt_begin_dev, gt_box_dev, gt_difficult_dev, det_pair_dev, det_box_dev,
                     workspace_dev, outcome_out_dev, (cudaStream_t)stream);
}

size_t b200_box_proposal_match_workspace_bytes(int num_props, int num_gt, int num_areas, int num_limits) {
    return box_proposal_match_workspace_bytes(num_props, num_gt, num_areas, num_limits);
}

int b200_box_proposal_match(int num_images, int num_props, int num_gt, int num_areas, int num_limits, int num_thresholds,
                            const float* prop_box_dev, const int* prop_begin_dev, const float* gt_box_dev, const double* gt_area_dev,
                            const int* gt_begin_dev, const int* prop_count_dev, const double* area_range_host, const double* thresholds_dev,
                            void* workspace, size_t workspace_bytes, float* overlap_out_dev, unsigned char* excluded_out_dev,
                            unsigned char* error_out_dev, long long* count_out_dev, b200_stream_t stream) {
    return box_proposal_match(num_images, num_props, num_gt, num_areas, num_limits, num_thresholds, prop_box_dev, prop_begin_dev, gt_box_dev,
                              gt_area_dev, gt_begin_dev, prop_count_dev, area_range_host, thresholds_dev, workspace, workspace_bytes,
                              overlap_out_dev, excluded_out_dev, error_out_dev, count_out_dev, (cudaStream_t)stream);
}

}  // extern "C"
