/*
 * b200_roi_ops.h -- C ABI of libb200_roi_ops.so: hand-written sm_90a CUDA replacements for the
 * per-image detection hot path of roytseng-tw/Detectron.pytorch (RoIAlign fwd/bwd in both
 * flavours, RoIPool, RoICrop, proposal NMS).
 *
 * The boundary mirrors the raw-pointer `extern "C"` launchers that sit under the reference's
 * cffi/THC glue (the layer its `_ext` modules bind): plain device pointers, ints and floats, a
 * CUDA stream, no torch types.  Each entry point cites the reference launcher it replaces
 * (paths relative to the reference repository root).
 *
 * Conventions (all entry points)
 *   - every pointer is a DEVICE pointer to dense, row-major ("contiguous") memory;
 *   - features / gradients are fp32 NCHW; rois are fp32 (R,5) = [batch_idx, x1, y1, x2, y2] in
 *     image pixels; boxes for NMS are fp32 (N,dim>=4) = [x1, y1, x2, y2, ...];
 *   - work is enqueued on `stream` (pass torch's current stream); calls never synchronise unless
 *     stated, keep no reference to caller memory after the enqueued work finishes, and are
 *     re-entrant per device;
 *   - outputs need NOT be pre-zeroed by the caller (the reference required `.zero_()`,
 *     functions/roi_align.py:23,39-40): every call fully defines its output;
 *   - return value: 0 = success; > 0 = a cudaError_t raised by the launch; < 0 = argument error
 *     (B200_ROI_EINVAL, B200_ROI_EWORKSPACE).  The reference instead returned 1/0 and called
 *     exit(-1) on a launch error (roi_align_kernel.cu:135-139); the Python layer turns a non-zero
 *     status into RuntimeError.
 */
#ifndef B200_ROI_OPS_H_
#define B200_ROI_OPS_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* b200_stream_t; /* == cudaStream_t */

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

#define B200_ROI_OK 0
#define B200_ROI_EINVAL (-1)
#define B200_ROI_EWORKSPACE (-2)

/* ABI version of this header (bumped on any signature change). */
B200_API int b200_roi_ops_abi_version(void);
/* Human-readable message for a status returned by any entry point. */
B200_API const char* b200_roi_ops_strerror(int status);

/* ---- RoIAlign, Caffe2/Detectron-exact variant (sampling_ratio) ---------------------------------
 * replaces ROIAlignForwardLaucher / ROIAlignBackwardLaucher,
 *   lib/modeling/roi_xfrom/roi_align/src/roi_align_kernel.cu:123-142, 272-290
 *   (declared lib/modeling/roi_xfrom/roi_align/src/roi_align_kernel.h:13-27; bound through
 *    roi_align_forward_cuda / roi_align_backward_cuda, src/roi_align_cuda.c:7-40, 42-76).
 * Same argument meaning and order; `batch_size` is added to the forward (the reference only passed
 * it to the backward) so that batch indices can be range-checked by the planner.
 * top: (R, C, aligned_height, aligned_width).  bottom_diff: (batch_size, C, H, W), fully written. */
B200_API int b200_roi_align_forward(const float* bottom_data, float spatial_scale, int batch_size, int num_rois,
                           int height, int width, int channels, int aligned_height, int aligned_width,
                           int sampling_ratio, const float* bottom_rois, float* top_data,
                           b200_stream_t stream);
B200_API int b200_roi_align_backward(const float* top_diff, float spatial_scale, int batch_size, int num_rois,
                            int height, int width, int channels, int aligned_height, int aligned_width,
                            int sampling_ratio, const float* bottom_rois, float* bottom_diff,
                            b200_stream_t stream);

/* Workspace variant of the forward: the feature-map-stationary fast path needs
 * b200_roi_align_workspace_bytes(batch_size, num_rois, height, width, aligned_height, aligned_width,
 * sampling_ratio) bytes of device scratch (per-RoI sample tables + per-tile RoI lists; 256-byte
 * aligned; 0 = fast path not applicable to these parameters).  The Python layer takes it from torch's caching allocator.  The plain
 * b200_roi_align_forward obtains the same scratch with cudaMallocAsync/cudaFreeAsync on `stream`.
 * With workspace == NULL (or too small) the shape-generic kernel runs.  Results are identical
 * either way up to ~1 ulp on bins whose samples straddle two tiles. */
B200_API size_t b200_roi_align_workspace_bytes(int batch_size, int num_rois, int height, int width,
                                               int aligned_height, int aligned_width, int sampling_ratio);
B200_API int b200_roi_align_forward_ws(const float* bottom_data, float spatial_scale, int batch_size, int num_rois,
                              int height, int width, int channels, int aligned_height, int aligned_width,
                              int sampling_ratio, const float* bottom_rois, float* top_data,
                              void* workspace, size_t workspace_bytes, b200_stream_t stream);

/* Workspace variant of the backward.  The fast paths need device scratch:
 *   - row-stationary gather path (no atomics): per-RoI tables, row-bucketed unit lists and a channel-innermost
 *     copy of dY (~ sizeof dY);
 *   - vector-reduction path: a channel-innermost scratch image of dX (= sizeof dX).
 * b200_roi_align_backward_workspace_bytes(...) returns what the path chosen for these parameters needs (0: the
 * scalar-atomic kernel runs and needs none).  NULL / too small -> the scalar-atomic kernel runs.  The plain
 * b200_roi_align_backward obtains the scratch with cudaMallocAsync/cudaFreeAsync on `stream`. */
B200_API size_t b200_roi_align_backward_workspace_bytes(int batch_size, int num_rois, int channels, int height, int width,
                                                        int aligned_height, int aligned_width, int sampling_ratio);
B200_API int b200_roi_align_backward_ws(const float* top_diff, float spatial_scale, int batch_size, int num_rois,
                               int height, int width, int channels, int aligned_height, int aligned_width,
                               int sampling_ratio, const float* bottom_rois, float* bottom_diff,
                               void* workspace, size_t workspace_bytes, b200_stream_t stream);

/* Indexed variants (SURVEY.md 8f N2: the FPN per-level loop + torch.cat + restore gather of
 * Generalized_RCNN.roi_feature_transform, lib/modeling/model_builder.py:264-303): RoI r reads / writes row
 * top_rows[r] of top_data / top_diff instead of row r, so the pooled features of every pyramid level land directly
 * in the restored order of one shared output tensor (and the backward picks its gradient rows out of the shared
 * tensor) -- no concatenated intermediate, no gather pass.  top_rows == NULL is the identity (= the _ws variants).
 * The forward writes exactly the rows named by top_rows; the caller sizes top_data. */
B200_API int b200_roi_align_forward_indexed(const float* bottom_data, float spatial_scale, int batch_size, int num_rois,
                                   int height, int width, int channels, int aligned_height, int aligned_width,
                                   int sampling_ratio, const float* bottom_rois, const int* top_rows, float* top_data,
                                   void* workspace, size_t workspace_bytes, b200_stream_t stream);
B200_API int b200_roi_align_backward_indexed(const float* top_diff, const int* top_rows, float spatial_scale, int batch_size,
                                    int num_rois, int height, int width, int channels, int aligned_height,
                                    int aligned_width, int sampling_ratio, const float* bottom_rois, float* bottom_diff,
                                    void* workspace, size_t workspace_bytes, b200_stream_t stream);

/* ---- RoIAlign, legacy variant (one bilinear sample per lattice corner, fp64 interpolation) -----
 * replaces ROIAlignForwardLaucher / ROIAlignBackwardLaucher,
 *   lib/model/roi_align/src/roi_align_kernel.cu:73-91, 145-162 (header roi_align_kernel.h). */
B200_API int b200_roi_align_legacy_forward(const float* bottom_data, float spatial_scale, int batch_size, int num_rois,
                                  int height, int width, int channels, int aligned_height, int aligned_width,
                                  const float* bottom_rois, float* top_data, b200_stream_t stream);
B200_API int b200_roi_align_legacy_backward(const float* top_diff, float spatial_scale, int batch_size, int num_rois,
                                   int height, int width, int channels, int aligned_height, int aligned_width,
                                   const float* bottom_rois, float* bottom_diff, b200_stream_t stream);

/* ---- RoIPool -----------------------------------------------------------------------------------
 * replaces ROIPoolForwardLaucher / ROIPoolBackwardLaucher,
 *   lib/model/roi_pooling/src/roi_pooling_kernel.cu:95-125, 205-234 (header roi_pooling_kernel.h:8-18).
 * argmax_data: int32 (R, C, PH, PW), flat index into the WHOLE bottom tensor or -1; may be NULL in
 * the forward.  The backward is deterministic and bit-identical to the reference's gather. */
B200_API int b200_roi_pool_forward(const float* bottom_data, float spatial_scale, int batch_size, int num_rois,
                          int height, int width, int channels, int pooled_height, int pooled_width,
                          const float* bottom_rois, float* top_data, int* argmax_data, b200_stream_t stream);
B200_API int b200_roi_pool_backward(const float* top_diff, float spatial_scale, int batch_size, int num_rois,
                           int height, int width, int channels, int pooled_height, int pooled_width,
                           const float* bottom_rois, float* bottom_diff, const int* argmax_data,
                           b200_stream_t stream);

/* ---- RoICrop (bilinear sampler from an explicit grid) -----------------------------------------
 * replaces BilinearSamplerBHWD_updateOutput_cuda_kernel / _updateGradInput_cuda_kernel,
 *   lib/model/roi_crop/src/roi_crop_cuda_kernel.cu:201-255, 257-326 (header roi_crop_cuda_kernel.h:6-32).
 * image: (N, C, H, W); grids: (R, out_h, out_w, 2) with channel 0 = y, channel 1 = x in [-1, 1];
 * output: (R, C, out_h, out_w).  RoI b samples image b / (R / N) (kernel :64, :217).  Dense tensors
 * only (the reference took explicit strides; the Python layer makes inputs contiguous).
 * grad_grids (same shape as grids) is zero-filled when non-NULL: the reference CUDA kernel never
 * stores the grid gradient (:111-194), so the observable result is zeros. */
B200_API int b200_roi_crop_forward(const float* image, const float* grids, int batch_size, int channels, int height,
                          int width, int num_rois, int out_height, int out_width, float* output,
                          b200_stream_t stream);
B200_API int b200_roi_crop_backward(const float* grad_output, const float* grids, int batch_size, int channels,
                           int height, int width, int num_rois, int out_height, int out_width,
                           float* grad_image, float* grad_grids, b200_stream_t stream);
/* Same with caller-supplied scratch (the Python layer takes it from torch's caching allocator): when the image gradient goes
 * through the channel-innermost scratch image (vector reductions; C % 4 == 0 and enough taps) it needs
 * b200_roi_crop_backward_workspace_bytes() bytes -- 0 when the scalar-atomic kernel is used.  b200_roi_crop_backward obtains
 * the scratch with cudaMallocAsync / cudaFreeAsync on `stream`. */
B200_API size_t b200_roi_crop_backward_workspace_bytes(int batch_size, int channels, int height, int width, int num_rois,
                                                       int out_height, int out_width);
B200_API int b200_roi_crop_backward_ws(const float* grad_output, const float* grids, int batch_size, int channels, int height,
                                       int width, int num_rois, int out_height, int out_width, float* grad_image,
                                       float* grad_grids, void* workspace, size_t workspace_bytes, b200_stream_t stream);

/* ---- proposal NMS ------------------------------------------------------------------------------
 * replaces nms_cuda_compute, lib/model/nms/src/nms_cuda_kernel.cu:87-161 (header nms_cuda_kernel.h:5-6;
 * bound through nms_cuda, src/nms_cuda.c:8-19).
 * boxes_dev: (boxes_num, boxes_dim) fp32, ALREADY sorted by score (the function never sorts).
 * keep_out_dev: int32[boxes_num], receives the kept row indices in ascending order;
 * num_out_dev: int32[1], receives their count.  Unlike the reference (cudaMalloc/cudaFree, four
 * blocking memcpys, host-side greedy scan, legacy default stream) everything runs on `stream` with
 * no host round trip; scratch comes from the caller: `workspace` must hold at least
 * b200_nms_workspace_bytes(boxes_num) bytes (256-byte aligned). */
B200_API size_t b200_nms_workspace_bytes(int boxes_num);
B200_API int b200_nms(const float* boxes_dev, int boxes_num, int boxes_dim, float nms_overlap_thresh,
             int* keep_out_dev, int* num_out_dev, void* workspace, size_t workspace_bytes,
             b200_stream_t stream);

/* ---- RoIAlign over a feature pyramid in ONE launch sequence (SURVEY.md 8f N2) -------------------------------------
 * replaces the per-level loop + torch.cat + gather of Generalized_RCNN.roi_feature_transform,
 * lib/modeling/model_builder.py:264-303: `num_levels` feature maps (same batch size and channel count, any H x W), the
 * RoIs of all levels stored level-major in bottom_rois (level l owns rows level_roi_begin_host[l] .. [l + 1]), and
 * top_rows[r] = the row of top_data RoI r is written to (the inverse of the reference's restore permutation; NULL:
 * identity).  The four *_host arrays and bottom_data_host (device pointers of the maps) are HOST arrays read during the
 * call.  The quad-strip kernel walks the strip columns of every level; results are bit-identical to per-level
 * b200_roi_align_forward calls.  b200_roi_align_fpn_workspace_bytes(...) == 0 means "not applicable" (sampling_ratio
 * outside {1, 2}, too many strip columns, B200_ROI_ALIGN_PATH other than auto or quad): loop over
 * b200_roi_align_forward_indexed instead; b200_roi_align_forward_fpn then returns B200_ROI_EWORKSPACE. */
B200_API size_t b200_roi_align_fpn_workspace_bytes(int num_levels, const int* heights_host, const int* widths_host,
                                                   int batch_size, int num_rois, int aligned_height, int aligned_width,
                                                   int sampling_ratio);
B200_API int b200_roi_align_forward_fpn(int num_levels, const float* const* bottom_data_host, const int* heights_host,
                                        const int* widths_host, const float* spatial_scales_host,
                                        const int* level_roi_begin_host, int batch_size, int num_rois, int channels,
                                        int aligned_height, int aligned_width, int sampling_ratio,
                                        const float* bottom_rois, const int* top_rows, float* top_data, void* workspace,
                                        size_t workspace_bytes, b200_stream_t stream);

/* Several independent NMS problems in ONE pair of launches (mask kernel over all problems' tiles, one scan CTA per
 * problem): the (image, FPN level) proposal sets of one step (lib/modeling/generate_proposals.py:91-99 runs them one
 * after the other on the host).  Problem p has counts_host[p] score-sorted rows, stored back to back in boxes_dev;
 * its kept indices (relative to its own first row) go to keep_out_dev + (sum of the counts before p), their number to
 * num_out_dev[p].  counts_host is a HOST array (the counts are launch geometry); 1 <= num_problems <= 64 and every
 * count <= ~13 800 (the pipelined scan's shared-memory limit), else B200_ROI_EINVAL -- loop over b200_nms then.
 * Results per problem are bit-identical to b200_nms. */
B200_API size_t b200_nms_batched_workspace_bytes(const int* counts_host, int num_problems);
B200_API int b200_nms_batched(const float* boxes_dev, const int* counts_host, int num_problems, int boxes_dim,
                              float nms_overlap_thresh, int* keep_out_dev, int* num_out_dev, void* workspace,
                              size_t workspace_bytes, b200_stream_t stream);
/* The same with the IoU test of the reference's Cython NMS (lib/utils/cython_nms.pyx:37-87), which its test-time
 * post-processing calls per class: both box areas rounded on their own, IoU = inter / ((Sa + Sb) - inter), suppress on
 * IoU >= thresh (b200_nms / b200_nms_batched: the reference CUDA kernel's fused area and IoU > thresh).  The kept indices
 * are those of cython_nms.nms on the same score-sorted rows.  Workspace: b200_nms_batched_workspace_bytes. */
B200_API int b200_nms_batched_cython(const float* boxes_dev, const int* counts_host, int num_problems, int boxes_dim,
                                     float nms_overlap_thresh, int* keep_out_dev, int* num_out_dev, void* workspace,
                                     size_t workspace_bytes, b200_stream_t stream);

/* ---- test-time detection post-processing (SURVEY.md 8f N3) ------------------------------------------------------
 * The per-class problems of lib/core/test.py:732-790 (box_results_with_nms_and_limit), batched like b200_nms_batched:
 * problem p = the detections of one class, counts_host[p] rows of [x1, y1, x2, y2, score] stored back to back
 * (1 <= num_problems <= 128).  Classic NMS goes through b200_nms_batched_cython.
 * b200_soft_nms_batched: lib/utils/cython_nms.pyx:98-203 step for step (method 1 linear, 2 gaussian, else hard), IN PLACE:
 *   afterwards problem p's first num_out_dev[p] rows are its surviving detections with decayed scores, in the
 *   reference's output order, and inds_out_dev holds their original row indices (relative to the problem).
 * b200_box_voting_batched: lib/utils/boxes.py:268-317; top_dets (the NMS survivors) are replaced in out_dev by the
 *   score-weighted average of all_dets rows with IoU >= thresh (cython_bbox.bbox_overlaps convention); scoring_method
 *   0 ID, 1 AVG, 2 IOU_AVG, 3 TEMP_AVG, 4 GENERALIZED_AVG, 5 QUASI_SUM. */
B200_API int b200_soft_nms_batched(float* dets_dev, const int* counts_host, int num_problems, float sigma, float overlap_thresh,
                                   float score_thresh, int method, int* inds_out_dev, int* num_out_dev, b200_stream_t stream);
B200_API int b200_box_voting_batched(const float* top_dets_dev, const int* top_counts_host, const float* all_dets_dev,
                                     const int* all_counts_host, int num_problems, float thresh, int scoring_method, float beta,
                                     float* out_dev, b200_stream_t stream);

/* ---- test-time mask paste + COCO RLE (SURVEY.md 8f N3, lib/core/test.py:793-847) ---------------------------------
 * The loop body of segm_results for the D detections of one image: box expanded by (M + 2) / M in float32 and truncated
 * to int32, M x M soft mask zero-padded and resized to the box with cv2.resize's float32 INTER_LINEAR arithmetic (IPP
 * off; 2x shrinks on both axes are cv2's INTER_AREA), thresholded with `> thresh`, pasted into an im_h x im_w image.
 *   masks_dev       float32 (D, num_channels, M, M), dense;
 *   mask_class_dev  int32 (D,): the channel detection d reads (a value outside [0, num_channels) reads as all zeros);
 *   boxes_dev       float32 (D, 4) = [x1, y1, x2, y2], not yet expanded.
 * A box whose expanded box lies wholly outside the image gives an empty mask (one count, im_h * im_w); non-finite boxes
 * do not fault, their result is unspecified.  1 <= M <= 64, im_h * im_w < 2^28, else B200_ROI_EINVAL.
 * COCO RLE of each detection's full-image mask (pycocotools mask.encode + rleToString), in two launches whatever D is:
 *   b200_segm_rle_sizes  writes sizes_out_dev int32 (D, 2) = [number of counts, string bytes] and leaves its scan state
 *                        in `workspace` (b200_segm_workspace_bytes(D) bytes, host arithmetic; else B200_ROI_EWORKSPACE);
 *   b200_segm_rle_emit   same inputs, the sizes and the workspace of that call: counts_out_dev int32 (sum of counts):
 *                        column-major run lengths starting with a run of zeros, summing to im_h * im_w per detection;
 *                        strings_out_dev (sum of bytes): the compressed COCO strings, no terminators; count_offsets /
 *                        string_offsets int64 (D + 1): where detection d's counts and string start.
 * The caller reads the sizes once to allocate the outputs.
 * b200_paste_masks: the full-image masks themselves, uint8 (D, im_h, im_w) (D <= 65535), the reference's im_mask. */
B200_API size_t b200_segm_workspace_bytes(int num_dets);
B200_API int b200_segm_rle_sizes(const float* masks_dev, const int* mask_class_dev, const float* boxes_dev, int num_dets, int num_channels,
                                 int resolution, int im_h, int im_w, float thresh, int* sizes_out_dev, void* workspace,
                                 size_t workspace_bytes, b200_stream_t stream);
B200_API int b200_segm_rle_emit(const float* masks_dev, const int* mask_class_dev, const float* boxes_dev, int num_dets, int num_channels,
                                int resolution, int im_h, int im_w, float thresh, const int* sizes_dev, const void* workspace,
                                size_t workspace_bytes, int* counts_out_dev, long long* count_offsets_out_dev,
                                unsigned char* strings_out_dev, long long* string_offsets_out_dev, b200_stream_t stream);
B200_API int b200_paste_masks(const float* masks_dev, const int* mask_class_dev, const float* boxes_dev, int num_dets, int num_channels,
                              int resolution, int im_h, int im_w, float thresh, unsigned char* out_dev, b200_stream_t stream);

/* ---- test-time keypoint extraction + OKS NMS (SURVEY.md 8f N3, lib/utils/keypoints.py:103-157, 225-266) -----------
 * b200_heatmaps_to_keypoints: heatmaps_to_keypoints for the D detections of one image, one launch.
 *   maps_dev      float32 (D, K, M, M), dense: the keypoint head's logits;
 *   rois_dev      float32 (D, 4) = [x1, y1, x2, y2];
 *   xy_preds_dev  float32 (D, 4, K): rows x, y, logit, prob.
 * Each heatmap is resized to max(ceil(max(x2 - x1, 1)), min_size) x ... pixels (min_size <= 0: no minimum) with
 * cv2.resize's float32 INTER_CUBIC arithmetic on the K-channel image; x, y are the box coordinates of the first maximum
 * (row-major), logit its value, prob the spatial softmax there (the sum of exponentials is accumulated in double).
 * The resized maps are never stored.  A side above 16384 pixels, or a non-finite box, is resized to 16384 pixels (the
 * reference would build that map); non-finite logits give an unspecified result.  1 <= M <= 64, K >= 1,
 * min_size <= 16384, D * K < 2^31, else B200_ROI_EINVAL.
 * b200_nms_oks: the greedy OKS NMS of nms_oks on those predictions (K must be 17, the COCO keypoints; D <= 4096), one
 * single-CTA launch.  Score = float32 mean of the 17 logits; descending score, equal scores the higher index first; OKS
 * in float64 with the COCO sigmas and the area (x2 - x1 + 1)(y2 - y1 + 1); a candidate is dropped when OKS > thresh.
 * Writes the kept indices in greedy order to keep_dev int32 (D,) and their number to num_keep_dev int32 (1,).
 * D == 0: both return B200_ROI_OK without writing anything. */
B200_API int b200_heatmaps_to_keypoints(const float* maps_dev, const float* rois_dev, int num_rois, int num_keypoints, int heatmap_size,
                                        int min_size, float* xy_preds_dev, b200_stream_t stream);
B200_API int b200_nms_oks(const float* xy_preds_dev, const float* rois_dev, int num_rois, int num_keypoints, double thresh, int* keep_dev,
                          int* num_keep_dev, b200_stream_t stream);

/* ---- introspection used by the benchmark / tests (no compute) ----------------------------------
 * Number of kernel launches the library has enqueued since load (all entry points). */
B200_API unsigned long long b200_roi_ops_launch_count(void);
/* Path-selection switches (A/B runs and tests reach paths the dispatch otherwise picks by shape): name is one of
 * "B200_ROI_ALIGN_PATH" (auto|generic|tiled|stream|quad), "B200_ROI_ALIGN_BWD_PATH" (auto|generic|nhwc|rows),
 * "B200_ROI_ALIGN_BWD_CPL" (4|2), "B200_NMS_SCAN" (resolver|simple);
 * value NULL or "" restores the default.  Each switch takes its initial value from the
 * environment variable of the same name, read once at first use -- no entry point calls getenv() on the hot path.
 * Returns 0, or B200_ROI_EINVAL for an unknown name. */
B200_API int b200_roi_ops_set_option(const char* name, const char* value);
/* Debug: register (or clear with NULL) one buffer with two uses.  The NMS kernels add their phase clock deltas to its
 * first 16 uint64 words.  The two streaming RoIAlign forwards write a watchdog record into [CTA][32] uint64 (one word per
 * warp) when a wait has spun half way to its trap; host-pinned memory keeps those records readable after the trap. */
B200_API void b200_roi_ops_debug_timing_buffer(void* device_u64x16);

/* ---- RPN proposal decode (SURVEY.md 8f N1: the GPU-resident proposal layer) --------------------------------
 * replaces the numpy block of GenerateProposalsOp.proposals_for_one_image, lib/modeling/generate_proposals.py:108-150
 * (gather by score order, utils.boxes.bbox_transform :157-196, clip_tiled_boxes :138-154, _filter_boxes :171-182),
 * for candidates that were selected and sorted on the device.  `order` holds indices into the (H, W, A)-flattened
 * score map, best first; row t of dets_out is (x1, y1, x2, y2, score) ready for b200_nms, or the degenerate box
 * (0, 0, -1, -1, score) with valid_out[t] = 0 when the size / centre filter rejects the candidate (such rows cannot
 * interact with any box in NMS; the caller drops them afterwards).  min_size is already multiplied by im_info[2]. */
B200_API int b200_proposal_decode(const float* bbox_deltas, const float* anchors, const long long* order, const float* scores,
                         int num_candidates, int num_anchors, int height, int width, float feat_stride, float im_height,
                         float im_width, float min_size, float* dets_out, int* valid_out, b200_stream_t stream);

/* ---- batched top-k of RPN score maps (SURVEY.md 8f N1) ----------------------------------------------------------
 * replaces np.argpartition + np.argsort of lib/modeling/generate_proposals.py:118-131 (and the torch.topk / torch.sort the
 * first device version used): problem p is one (A_p, H_p * W_p) float32 score map on the device, read where it lies;
 * order_out receives, best first, the k_p indices into its (H, W, A) flattening (what b200_proposal_decode takes as
 * `order`), scores_out the scores; problems are stored back to back.  <= 64 problems, k_p <= 16384 (else
 * B200_ROI_EWORKSPACE: the caller sorts by other means).  Equal scores come out in ascending index; which of several
 * scores EQUAL TO THE k-th are taken is deterministic (memory order), the reference leaves it unspecified.
 * Radix select (3 histogram launches, chunk-parallel) + one collect-and-sort launch; no host read. */
B200_API size_t b200_topk_batched_workspace_bytes(int num_problems);
B200_API int b200_topk_batched(const float* const* scores_dev_ptrs_host, const int* num_anchors_host, const int* num_cells_host,
                               const int* k_host, int num_problems, long long* order_out_dev, float* scores_out_dev, void* workspace,
                               size_t workspace_bytes, b200_stream_t stream);

/* ---- RoI label / regression-target generation on the device (SURVEY.md 8f N4) ---------------------------------
 * The per-image host work of the reference's training data path, for proposals that already live on the GPU.  Boxes are
 * float32 (x1, y1, x2, y2) rows in image pixels, exactly the roidb's `boxes`.
 * b200_bbox_overlaps    lib/utils/cython_bbox.pyx:32-73: (N, K) IoU with the +1 pixel convention, bit-exact float32.
 * b200_roi_assign       lib/datasets/json_dataset.py:429-463 + :514-531 without the (N, K) matrix: per box the best
 *                       ground-truth overlap (0 when none is positive), its index (first maximum; -1) and class (0).
 * b200_roi_select       lib/roi_data/fast_rcnn.py:138-151: ascending index lists of the foreground (>= fg_thresh) and
 *                       background ([bg_lo, bg_hi)) boxes, counts_out = {num_fg, num_bg}.
 * b200_fast_rcnn_targets  fast_rcnn.py:161-187 + :203-248 for the kept rows (the first num_fg are foreground): labels
 *                       (int32), rois (batch_idx, box * im_scale), regression targets (utils/boxes.py:199-230) expanded
 *                       to 4 * num_reg_classes columns, inside / outside weights.  bbox_reg_weights_host: 4 floats. */
B200_API int b200_bbox_overlaps(const float* boxes_dev, int num_boxes, const float* query_boxes_dev, int num_query,
                                float* overlaps_out_dev, b200_stream_t stream);
B200_API int b200_roi_assign(const float* boxes_dev, int num_boxes, const float* gt_boxes_dev, const int* gt_classes_dev, int num_gt,
                             float* max_overlaps_out_dev, int* argmax_out_dev, int* max_classes_out_dev, b200_stream_t stream);
B200_API int b200_roi_select(const float* max_overlaps_dev, int num_boxes, float fg_thresh, float bg_thresh_hi, float bg_thresh_lo,
                             int* fg_inds_out_dev, int* bg_inds_out_dev, int* counts_out_dev, b200_stream_t stream);
B200_API int b200_fast_rcnn_targets(const float* boxes_dev, const float* gt_boxes_dev, const int* argmax_dev, const int* max_classes_dev,
                                    const int* keep_inds_dev, int num_keep, int num_fg, const float* bbox_reg_weights_host,
                                    int num_reg_classes, int cls_agnostic, float im_scale, float batch_idx, int* labels_out_dev,
                                    float* rois_out_dev, float* bbox_targets_out_dev, float* inside_weights_out_dev,
                                    float* outside_weights_out_dev, b200_stream_t stream);

/* ---- RPN anchor labels and box-regression targets (training, lib/roi_data/rpn.py:40-261) -------------------------------
 * add_rpn_blobs / _get_rpn_blobs for all images and all anchor levels of a step, in a fixed number of launches.
 * Level table (HOST arrays, 1 <= num_levels <= 8): field_sizes_host[l] = F_l, num_cell_anchors_host[l] = A_l (sum <= 32),
 *   strides_host[l], cell_anchors_host (sum A_l, 4) float64 = generate_anchors(stride_l, sizes_l, ratios).  Anchor i of the
 *   call is the reference's concatenated order: level, then (h, w, a); it is float32(cell anchor + (w, h, w, h) * stride), the
 *   rounding of data_utils.py:69-93, computed where it is needed.
 * Image table (HOST arrays, 1 <= num_images <= 64): im_sizes_host (N, 2) float64 = (im_height, im_width); image n's ground
 *   truth is rows gt_begin_host[n] .. gt_begin_host[n + 1] - 1 of gt_boxes_dev (float32 (x1, y1, x2, y2), already scaled), and
 *   every image needs at least one (the reference fails without, rpn.py:144-186).
 * b200_rpn_labels  rpn.py:115-170 + the candidate sets of :174 / :186: inside test (straddle_thresh < 0 keeps every anchor;
 *   x1, y1 >= float32(-straddle), x2 < im_width + straddle and y2 < im_height + straddle in float64), IoU with
 *   cython_bbox.bbox_overlaps' arithmetic, fg candidates = anchors whose row equals some ground-truth box's maximum over the
 *   inside anchors or whose row maximum is >= positive_overlap, bg candidates = row maximum < negative_overlap (fg included).
 *   counts_out_dev int32 (N, 3) = (#fg candidates, #bg candidates, #inside anchors).  memset + 3 launches.
 * The caller reads the counts once and draws: per image, positions into the ascending fg candidate list to disable
 *   (npr.choice(fg_inds, #fg - num_fg, replace=False), rpn.py:175-179) and positions into the ascending bg candidate list to
 *   enable (npr.randint(#bg, size=num_bg), :185-189, only when #bg > num_bg).
 * b200_rpn_emit  rpn.py:176-259 with that draw: fg_disable_dev / bg_enable_dev int32, image n's positions at
 *   [*_begin_host[n], *_begin_host[n + 1]) (HOST tables, N + 1 entries; positions out of range are ignored).  Disables first,
 *   then enables; targets (utils/boxes.py:199-230, weights 1) for the fg set left by the disable draw, even where the enable
 *   draw relabels one of them 0; inside weights 1 where the final label is 1; outside weights float32(1.0 / #labels >= 0)
 *   where it is >= 0.  Writes EVERY element of level l's blobs, the four device pointers of the *_out_host tables:
 *   labels int32 (N, A_l, F_l, F_l), bbox targets / inside / outside weights float32 (N, 4 A_l, F_l, F_l); anchors outside
 *   the image get -1 / 0.  Blobs with F_l * F_l % 4 == 0 must be 16-byte aligned.  3 launches.
 * Both take the same tables, `counts_dev` is the labelling call's output, and the workspace (b200_rpn_targets_workspace_bytes
 * bytes, about 13 bytes per (image, anchor)) carries the labelling state to the emit call.  Bad sizes, tables or null pointers:
 * B200_ROI_EINVAL before any launch; a missing or small workspace: B200_ROI_EWORKSPACE. */
B200_API size_t b200_rpn_targets_workspace_bytes(int num_levels, const int* field_sizes_host, const int* num_cell_anchors_host, int num_images,
                                                 int num_gt_total);
B200_API int b200_rpn_labels(int num_levels, const int* field_sizes_host, const int* num_cell_anchors_host, const double* strides_host,
                             const double* cell_anchors_host, int num_images, const double* im_sizes_host, const int* gt_begin_host,
                             const float* gt_boxes_dev, double straddle_thresh, float positive_overlap, float negative_overlap,
                             int* counts_out_dev, void* workspace, size_t workspace_bytes, b200_stream_t stream);
B200_API int b200_rpn_emit(int num_levels, const int* field_sizes_host, const int* num_cell_anchors_host, const double* strides_host,
                           const double* cell_anchors_host, int num_images, const double* im_sizes_host, const int* gt_begin_host,
                           const float* gt_boxes_dev, double straddle_thresh, const int* counts_dev, const int* fg_disable_dev,
                           const int* fg_disable_begin_host, const int* bg_enable_dev, const int* bg_enable_begin_host, void* workspace,
                           size_t workspace_bytes, int* const* labels_out_host, float* const* bbox_targets_out_host,
                           float* const* inside_weights_out_host, float* const* outside_weights_out_host, b200_stream_t stream);

/* ---- Mask R-CNN mask targets (training, lib/roi_data/mask_rcnn.py:34-122 with lib/utils/segms.py:93-131) -------------------
 * add_mask_rcnn_blobs' masks_int32 for all images of a step, in 2 launches whatever the image, RoI, object or vertex count.
 * RoIs: rois_dev (R, 4) float32 (x1, y1, x2, y2) in UNSCALED image coordinates (16-byte aligned), roi_image_dev (R,) int32
 *   image index, roi_class_dev (R,) int32 class; R >= 1.  A RoI with class <= 0 (the reference's empty-fg fallback row), with
 *   class >= num_classes (class-specific), or in an image without objects gets an all -1 row.
 * Objects (HOST table, 1 <= num_images <= 64): image n's non-crowd objects are obj_begin_host[n] .. obj_begin_host[n + 1] - 1
 *   (obj_begin_host[0] = 0, non-decreasing).  Object o's polygons are poly_begin_dev[o] .. poly_begin_dev[o + 1] - 1 (at least
 *   one), polygon p's coordinates coords_dev[coord_begin_dev[p] .. coord_begin_dev[p + 1]) as float32 x, y pairs, packed in
 *   order (coord_begin_dev[0] = 0, even, non-decreasing; num_polys + 1 and num_objects + 1 entries).  Coordinates must lie
 *   within +-2^20 so the upsampled positions stay in int32.
 * Per RoI with a class: the object whose tight polygon box (segms.py:120-131, written to obj_boxes_out_dev (num_objects, 4),
 *   16-byte aligned) has the first maximum cython_bbox IoU (mask_rcnn.py:57-64); its polygons normalised to the RoI in float32
 *   ((p - x1) * M / max(x2 - x1, 1), segms.py:104-110) and rasterised as pycocotools' rleFrPoly + decode on an M x M grid,
 *   union over the polygons (segms.py:112-117).
 * masks_out_dev int32 (R, num_classes * M * M), or (R, M * M) for num_classes = 0 (class-agnostic): the RoI's class slice
 *   holds the [y][x] mask (0 / 1), every other element -1 (mask_rcnn.py:108-122).  16-byte aligned when the row length is a
 *   multiple of 4.  1 <= resolution (M) <= 64.  Bad sizes, host tables or null pointers: B200_ROI_EINVAL before any launch. */
B200_API int b200_mask_targets(const float* rois_dev, const int* roi_image_dev, const int* roi_class_dev, int num_rois, int num_images,
                               const int* obj_begin_host, int num_polys, const int* poly_begin_dev, int num_coords, const int* coord_begin_dev,
                               const float* coords_dev, int resolution, int num_classes, float* obj_boxes_out_dev, int* masks_out_dev,
                               b200_stream_t stream);

/* ---- Keypoint R-CNN keypoint targets (training, lib/roi_data/keypoint_rcnn.py:33-82 with lib/utils/keypoints.py:160-211) ---
 * add_keypoint_rcnn_blobs for all images of a step in 2 launches (one per call) whatever the image, box or person count, with
 * the caller's draw in between.  Shared inputs (1 <= num_images <= 64, HOST tables starting at 0 and non-decreasing):
 *   boxes_dev (B, 4) float32 (x1, y1, x2, y2) UNSCALED, image n's merged roidb boxes in rows box_begin_host[n] .. [n + 1] - 1
 *   (ground truth first, then proposals; B <= 2^29); box_to_gt_dev (B,) int32 = roidb['box_to_gt_ind_map'] (an index into the
 *   image's gt_inds, numpy-style: -1 is the last entry; out of range: no person); gt_inds_dev = each image's
 *   np.where(gt_classes > 0), rows gt_begin_host[n] .. [n + 1] - 1, values indexing the image's keypoint rows;
 *   keypoints_dev (P, 3, K) int32 = every image's gt_keypoints (x, y, v rows), image n's in rows person_begin_host[n] .. [n + 1]
 *   - 1.  1 <= num_keypoints (K) <= 64.
 * b200_keypoint_candidates (keypoint_rcnn.py:37-51): box b of image n is a candidate when max_overlaps_dev[b] >= fg_thresh
 *   (float32) and its person has a keypoint with v > 0 inside the box, ends included, compared in double (_within_box).
 *   candidates_out_dev (B,) int32: image n's candidates as ascending image-relative box indices from row box_begin_host[n];
 *   counts_out_dev (N,) int32: their number per image.  Nothing else is written.
 * b200_keypoint_targets (keypoint_rcnn.py:59-82): image n's selected RoIs are rows roi_begin_host[n] .. [n + 1] - 1 (never more
 *   than the image's boxes); picks_dev[r] is the position of RoI r in its image's candidate list (< counts_dev[n], else the row
 *   is unspecified).  Per (RoI r, keypoint k), with the person's keypoints (all -1 when box_to_gt < 0), in float32:
 *   s = HS / (x2 - x1), floor((x - x1) * s), HS - 1 when x == x2 (the same for y); valid = 0 <= x, y < HS and v > 0;
 *   locations_out_dev[r * K + k] int32 = y * HS + x when valid, else 0, or INT_MIN where that product is not finite (numpy's
 *   astype(int32) of NaN); weights_out_dev[r * K + k] float32 = valid.  rois_out_dev (R, 5) float32 = batch_index_host[n], then
 *   the box times im_scales_host[n] (float32 multiply).  1 <= heatmap_size (HS) <= 4096, R * K < 2^31.  Every output element is
 *   written once; with R = 0 the launch writes nothing (the pointers must still be valid).
 * Bad sizes, host tables or null pointers: B200_ROI_EINVAL before any launch. */
B200_API int b200_keypoint_candidates(const float* boxes_dev, const float* max_overlaps_dev, const int* box_to_gt_dev, int num_images,
                                      const int* box_begin_host, const int* gt_inds_dev, const int* gt_begin_host, const int* keypoints_dev,
                                      const int* person_begin_host, int num_keypoints, float fg_thresh, int* candidates_out_dev,
                                      int* counts_out_dev, b200_stream_t stream);
B200_API int b200_keypoint_targets(const float* boxes_dev, const int* box_to_gt_dev, int num_images, const int* box_begin_host,
                                   const int* gt_inds_dev, const int* gt_begin_host, const int* keypoints_dev, const int* person_begin_host,
                                   int num_keypoints, int heatmap_size, const int* candidates_dev, const int* counts_dev,
                                   const int* picks_dev, const int* roi_begin_host, const float* im_scales_host,
                                   const float* batch_index_host, float* rois_out_dev, int* locations_out_dev, float* weights_out_dev,
                                   b200_stream_t stream);

/* ---- input image blob (lib/utils/blob.py:37-148, lib/roi_data/minibatch.py:47-79, lib/roi_data/loader.py:251-260) ----------
 * The network's `data` blob for all images of a call in ONE launch, whatever their number and sizes: per image the decoded
 * uint8 BGR image, optionally flipped (im[:, ::-1, :]), minus PIXEL_MEANS, resized like cv2.resize(fx = fy = im_scale,
 * INTER_LINEAR) with IPP off, zero-padded and transposed to NCHW.
 * Image i is described by descs_dev[i] (a DEVICE array of num_images entries, 1 <= num_images <= 65535):
 *   src_offset   byte offset of its first pixel from src_dev; pixel (y, x) channel c is src_dev[src_offset + y * row_pitch + 3 x + c];
 *   height, width  its size (>= 1); row_pitch >= 3 * width;
 *   out_h, out_w   the resized size, cv2's (rint(height * im_scale), rint(width * im_scale)), at most blob_h x blob_w;
 *   inv_scale    1 / im_scale in double (cv2's scale; 1.0 when the resized size equals the input size: cv2 copies);
 *   flipped      non-zero: read source column width - 1 - s where the unflipped image reads s;
 *   area2x       non-zero when inv_scale == 2.0 exactly: cv2's fast INTER_AREA path;
 *   slot         its index in the output batch.  The slots of the call must be 0 .. num_images - 1, each once.
 * mean_table_dev (3, 256) float32: channel c of a pixel of value v after `im -= PIXEL_MEANS` (numpy's float32(float64(v) - mean)).
 * out_dev (num_images, 3, blob_h, blob_w) float32: every element written once, 0 outside each image's out_h x out_w; 16-byte
 *   stores when blob_w % 4 == 0 and out_dev is 16-byte aligned.  blob_h * blob_w < 2^31.
 * Bad sizes or null pointers: B200_ROI_EINVAL before any launch (the descriptors live on the device and are not read by the host). */
typedef struct b200_image_blob_desc {
    long long src_offset;
    long long row_pitch;
    double inv_scale;
    int height, width;
    int out_h, out_w;
    int flipped, area2x;
    int slot, reserved;
} b200_image_blob_desc;

B200_API int b200_image_blob(const unsigned char* src_dev, const b200_image_blob_desc* descs_dev, int num_images, const float* mean_table_dev,
                             int blob_h, int blob_w, float* out_dev, b200_stream_t stream);

/* ---- COCO evaluation (lib/datasets/json_dataset_evaluator.py:38-233, 320-430 -> pycocotools COCOeval) --------------------
 * The device stages of COCOeval.evaluate() and accumulate() for one iouType.  Work is grouped per (image, category) pair; pairs
 * are ordered image-major.  Pair p owns detections pair_det_begin[p] .. [p + 1] - 1 (results order), ground truth
 * pair_gt_begin[p] .. [p + 1] - 1 (annotation order), entries pair_entry_begin[p] .. [p + 1] - 1 (min(D, maxDets[-1]) each)
 * and IoU rows pair_iou_begin[p] (int64, entries x ground truth, float64, row = entry).  All tables are DEVICE int32 unless
 * stated.  gt_flags: bit 0 iscrowd, bit 1 ignore (iscrowd, or num_keypoints == 0 for keypoints), bit 2 annotation id != 0.
 * b200_coco_rank        (computeIoU's / evaluateImg's mergesort on -score, cut to maxDets[-1]) writes entry r of pair p:
 *                       entry_det (detection index), entry_rank (r), entry_score (float64).
 * b200_coco_bbox_iou    (computeIoU, iouType 'bbox': maskApi bbIou) det_box / gt_box float64 (x, y, w, h), 16-byte aligned.
 * b200_coco_oks         (computeOks) det_kp / gt_kp float64 (n, 17, 3) (x, y, v), gt_box float64 (x, y, w, h), gt_area float64,
 *                       vars_host = (sigmas * 2) ** 2 (17 float64, HOST).  exp() is CUDA's, not numpy's: within a few ulp.
 * b200_coco_masks       (annToRLE, rleFrString, rleFrPoly, rleMerge) column-major bitmaps: slot s is words[slot_word[s] ..
 *                       slot_word[s + 1]) (int64 word offsets) of an image of slot_hw[s] = (h, w) int32 pairs.  Strings (compressed
 *                       COCO counts, str_bytes[str_begin[i] .. [i + 1]), int64 offsets), uncompressed counts (uint32,
 *                       cnt_begin int64) and polygons (float64 x, y; polygon i is vertices vtx_begin[i] .. [i + 1] - 1, at least 3,
 *                       |coordinate| <= 2^20) each toggle into their slot; mask m is the union of slots mask_slot_begin[m] ..
 *                       [m + 1] - 1 (same image size), left in its first slot.  words is zeroed here (num_words words).  Writes
 *                       mask_area (int64) and mask_range (int32 pairs: first and last non-zero word, (1, 0) when empty).
 *                       Counts must add up to h * w, as pycocotools assumes.
 * b200_coco_segm_iou    (computeIoU, iouType 'segm': rleIou) pairs pair_begin .. + num_pairs - 1; detection d is mask d - det0,
 *                       ground truth g is mask gt_mask0 + g - gt0 of the b200_coco_masks call.
 * b200_coco_match       (evaluateImg at maxDets[-1]) 1 <= T <= 16 thresholds and 1 <= A <= 8 area ranges (HOST float64, [lo, hi]
 *                       pairs), A * T <= 64, max_gt = the largest ground truth count of a pair (A * T * max_gt <= 200 KiB).
 *                       entry_flags (A, num_entries) uint32, zeroed by the caller: bit t = matched to a ground truth with a non-zero
 *                       id at threshold t, bit 16 + t = ignored.  npig (K, A), zeroed by the caller: += non-ignored ground truth;
 *                       pair_cat = the pair's category index.
 * b200_coco_accumulate  (accumulate) order = all entries sorted stably by category index, then descending score, so that ties keep
 *                       (image, rank) order; category k's are order[cat_entry_begin[k] .. [k + 1]), cat_pairs[k] = its number of
 *                       pairs.  max_dets_host (M ints, HOST), rec_thrs float64 (R).  precision / scores (T, R, K, A, M) and recall
 *                       (T, K, A, M) float64 must hold -1 on entry; the skipped (category, area) cells keep it.
 *                       max_cat_entries = the largest category's entry count, < 2^21 (HOST value: the scans pack three counts);
 *                       workspace: A * M * num_entries * 20 bytes, 8-byte aligned, else B200_ROI_EWORKSPACE.
 * Bad sizes or null pointers: B200_ROI_EINVAL before any launch. */
B200_API int b200_coco_rank(int num_pairs, const int* pair_det_begin_dev, const int* pair_entry_begin_dev, const double* det_score_dev,
                            int* entry_det_out_dev, int* entry_rank_out_dev, double* entry_score_out_dev, b200_stream_t stream);
B200_API int b200_coco_bbox_iou(int num_pairs, const int* pair_gt_begin_dev, const int* pair_entry_begin_dev, const long long* pair_iou_begin_dev,
                                const int* entry_det_dev, const double* det_box_dev, const double* gt_box_dev, const int* gt_flags_dev,
                                double* ious_out_dev, b200_stream_t stream);
B200_API int b200_coco_oks(int num_pairs, const double* vars_host, const int* pair_gt_begin_dev, const int* pair_entry_begin_dev,
                           const long long* pair_iou_begin_dev, const int* entry_det_dev, const double* det_kp_dev, const double* gt_kp_dev,
                           const double* gt_box_dev, const double* gt_area_dev, double* ious_out_dev, b200_stream_t stream);
B200_API int b200_coco_masks(unsigned* words_dev, long long num_words, int num_slots, const long long* slot_word_dev, const int* slot_hw_dev,
                             int num_strings, const int* str_slot_dev, const long long* str_begin_dev, const unsigned char* str_bytes_dev,
                             int num_counts, const int* cnt_slot_dev, const long long* cnt_begin_dev, const unsigned* counts_dev,
                             int num_polys, int num_vertices, const int* poly_slot_dev, const int* vtx_begin_dev, const double* xy_dev,
                             int num_masks, const int* mask_slot_begin_dev, long long* mask_area_out_dev, int* mask_range_out_dev,
                             b200_stream_t stream);
B200_API int b200_coco_segm_iou(int pair_begin, int num_pairs, const int* pair_gt_begin_dev, const int* pair_entry_begin_dev,
                                const long long* pair_iou_begin_dev, const int* entry_det_dev, int det0, int gt0, int gt_mask0,
                                const int* mask_slot_begin_dev, const long long* slot_word_dev, const int* slot_hw_dev,
                                const unsigned* words_dev, const long long* mask_area_dev, const int* mask_range_dev, const int* gt_flags_dev,
                                double* ious_out_dev, b200_stream_t stream);
B200_API int b200_coco_match(int num_pairs, int num_thresholds, const double* iou_thrs_host, int num_areas, const double* area_rng_host,
                             int max_gt, const int* pair_gt_begin_dev, const int* pair_entry_begin_dev, const long long* pair_iou_begin_dev,
                             const int* pair_cat_dev, const int* entry_det_dev, const double* det_area_dev, const double* gt_area_dev,
                             const int* gt_flags_dev, const double* ious_dev, int num_entries, unsigned* entry_flags_dev, int* npig_dev,
                             b200_stream_t stream);
B200_API int b200_coco_accumulate(int num_cats, int num_areas, int num_max_dets, int num_thresholds, int num_recall, const int* max_dets_host,
                                  const int* cat_entry_begin_dev, const int* cat_pairs_dev, const int* order_dev, const int* entry_rank_dev,
                                  const double* entry_score_dev, const unsigned* entry_flags_dev, int num_entries, int max_cat_entries,
                                  const int* npig_dev,
                                  const double* rec_thrs_dev, void* workspace, size_t workspace_bytes, double* precision_out_dev,
                                  double* recall_out_dev, double* scores_out_dev, b200_stream_t stream);

/* ---- PASCAL VOC evaluation (lib/datasets/voc_eval.py:86-223, the per-detection loop) ------------------------------------------
 * b200_voc_match marks each detection a true positive, a false positive or neither, as the reference's loop does.
 * Detections: num_dets rows of det_box_dev (float64 x1, y1, x2, y2, 16-byte aligned) and det_pair_dev (int32, in 0 .. num_pairs - 1,
 *   the detection's (class, image) pair).  Within one class the rows are in rank order (the caller's sort), so a row's index is its rank.
 * Ground truth: pair p owns rows pair_gt_begin_dev[p] .. [p + 1] - 1 (num_pairs + 1 non-decreasing int32, last = num_gt) of gt_box_dev
 *   (float64 x1, y1, x2, y2, 16-byte aligned) and gt_difficult_dev (uint8, non-zero = difficult).
 * Overlap in float64 without contraction: iw = max(min(x2) - max(x1) + 1, 0), ih likewise, inters = iw * ih,
 *   uni = (bw * bh + gw * gh) - inters, ov = inters / uni; jmax = numpy's argmax (first maximum; a NaN wins and fails the test).
 * outcome_out_dev (num_dets uint8): 1 = tp (ov > ovthresh, jmax not difficult, the lowest-ranked such detection of jmax), 2 = neither
 *   (ov > ovthresh and jmax difficult), 0 = fp (every other case, no ground truth of the pair included).
 * workspace_dev: num_gt ints (overwritten).
 * Bad sizes or null pointers: B200_ROI_EINVAL before any launch. */
B200_API int b200_voc_match(int num_dets, int num_pairs, int num_gt, double ovthresh, const int* pair_gt_begin_dev, const double* gt_box_dev,
                            const unsigned char* gt_difficult_dev, const int* det_pair_dev, const double* det_box_dev, int* workspace_dev,
                            unsigned char* outcome_out_dev, b200_stream_t stream);

/* ---- Proposal recall (lib/datasets/json_dataset_evaluator.py:236-317, evaluate_box_proposals' greedy assignment) ---------------
 * b200_box_proposal_match runs the reference's per-image assignment for every (limit l, area range a, image i) in one launch.
 * Proposals: image i owns rows prop_begin_dev[i] .. [i + 1] - 1 (num_images + 1 non-decreasing int32, last = num_props) of prop_box_dev
 *   (float32 x1, y1, x2, y2, 16-byte aligned).  prop_count_dev (num_limits x num_images int32): how many of them limit l keeps, clamped
 *   to [0, P_i] (the caller's len(boxes[:limit])).  An image with P_i == 0 is skipped, as the reference skips it.
 * Ground truth: image i owns rows gt_begin_dev[i] .. [i + 1] - 1 (last = num_gt) of gt_box_dev (float32, 16-byte aligned) and
 *   gt_area_dev (float64 seg_areas); only non-crowd foreground boxes belong here.  area_range_host: num_areas (1 .. 8) float64 pairs
 *   [lo, hi]; a gt is in range when lo <= area <= hi (a NaN area never is).
 * Matching, per item, over the kept proposals x the in-range gts, IoU by the reference's cython bbox_overlaps (float32 with double
 *   area sums): min(P, G) times, the gt whose best IoU over the unused proposals is largest (lowest gt row on ties) is matched to the
 *   first proposal reaching it; that IoU is recorded and both are used.
 * Outputs, per (l, a, gt row) at [(l * num_areas + a) * num_gt + row]: overlap_out_dev (float32) the recorded IoU, 0 if unmatched;
 *   excluded_out_dev (uint8) 1 when the gt is out of range or its image is skipped (not part of gt_overlaps), else 0.
 *   error_out_dev (num_limits x num_areas x num_images uint8): 1 when a NaN IoU lies in the item's matrix and the reference's
 *   `assert gt_ovr >= 0` would fail (only items with at least one iteration); the item's outputs are then unspecified.
 *   count_out_dev (num_limits x num_areas x num_thresholds int64, 8-byte aligned): the counted gts with float64(overlap) >=
 *   thresholds_dev[t] (float64), summed over the images without error.
 * workspace: b200_box_proposal_match_workspace_bytes(...) bytes, overwritten (small or missing: B200_ROI_EWORKSPACE).
 * Bad sizes or null pointers: B200_ROI_EINVAL before any launch.  Zero items (no images, areas or limits): 0, outputs untouched. */
#define B200_BOX_PROPOSAL_MAX_AREAS 8
B200_API size_t b200_box_proposal_match_workspace_bytes(int num_props, int num_gt, int num_areas, int num_limits);
B200_API int b200_box_proposal_match(int num_images, int num_props, int num_gt, int num_areas, int num_limits, int num_thresholds,
                                     const float* prop_box_dev, const int* prop_begin_dev, const float* gt_box_dev, const double* gt_area_dev,
                                     const int* gt_begin_dev, const int* prop_count_dev, const double* area_range_host,
                                     const double* thresholds_dev, void* workspace, size_t workspace_bytes, float* overlap_out_dev,
                                     unsigned char* excluded_out_dev, unsigned char* error_out_dev, long long* count_out_dev,
                                     b200_stream_t stream);

/* ---- Training losses: RPN (lib/modeling/rpn_heads.py:130-161, lib/modeling/FPN.py:422-466) and Fast R-CNN
 *      (lib/modeling/fast_rcnn_heads.py:50-68), with net_utils.smooth_l1_loss (lib/utils/net.py:15-32) ---------------------
 * Element terms use the reference expression's float32 operations in its order (no FMA contraction, no element skipped for a
 * zero weight: a non-finite prediction under a zero weight gives NaN as `0 * NaN` does there).  Sums are taken in float64, per
 * CTA and then over the CTAs in a fixed order; the last CTA finishes them (integer ticket), so the results are bit-identical
 * from run to run and no call reads the host.
 * workspace: b200_loss_workspace_bytes(num_levels) bytes (the Fast R-CNN loss: num_levels = 1).  It must be zero-filled
 *   before its first use and is left zero by every completed forward call; calls that may run concurrently need separate
 *   workspaces.  Small or missing: B200_ROI_EWORKSPACE.
 *
 * RPN, one descriptor per level (num_levels 1 .. B200_RPN_LOSS_MAX_LEVELS, HOST array):
 *   cls_logits (N, cls_channels, h, w) with cls_channels = A (activation 0, sigmoid) or 2A (activation 1, softmax: the pair
 *   (a, A + a) of image n, the reference's view(N, 2, A, h, w)); bbox_pred (N, 4A, hb, wb); labels_wide int32 (N, A, label_h,
 *   label_w) and the three float32 blobs (N, 4A, target_h, target_w), read in their [:h, :w] / [:hb, :wb] window in place.
 * b200_rpn_loss_forward  losses_out (num_levels, 2) = (loss_cls, loss_bbox) per level; divisor_out (num_levels,) the cls
 *   divisor: fixed_divisor when > 0 with activation 0 (FPN: RPN_BATCH_SIZE_PER_IM * IMS_PER_BATCH), else the count of labels
 *   >= 0 (sigmoid) or != -1 (softmax, ignore_index = -1); 0 / 0 gives NaN, as in the reference.  Sigmoid: sum of
 *   BCE-with-logits(x, float(label)) * (label >= 0).  Softmax: sum of -log_softmax at the label; a label other than -1, 0, 1
 *   adds NaN.  Box: smooth L1 with beta = 1/9 summed, / N.  One launch.
 * b200_rpn_loss_backward  writes every element of each level's cls_grad (shape of cls_logits) and bbox_grad (shape of bbox_pred)
 *   from grad_losses_dev (num_levels, 2) and the forward's divisor_dev.  One launch (none when every level is empty).
 * Bad sizes (a wide blob smaller than its prediction, cls_channels not A / 2A) or null pointers: B200_ROI_EINVAL before any
 * launch. */
#define B200_RPN_LOSS_MAX_LEVELS 8
typedef struct b200_rpn_loss_level {
    const float* cls_logits;
    const float* bbox_pred;
    const int* labels_wide;
    const float* bbox_targets_wide;
    const float* bbox_inside_wide;
    const float* bbox_outside_wide;
    float* cls_grad;              /* backward only */
    float* bbox_grad;             /* backward only */
    int num_images, num_anchors, cls_channels;
    int h, w, hb, wb;
    int label_h, label_w, target_h, target_w;
} b200_rpn_loss_level;

B200_API size_t b200_loss_workspace_bytes(int num_levels);
B200_API int b200_rpn_loss_forward(int num_levels, const b200_rpn_loss_level* levels_host, int activation, float fixed_divisor,
                                   void* workspace, size_t workspace_bytes, float* losses_out_dev, float* divisor_out_dev,
                                   b200_stream_t stream);
B200_API int b200_rpn_loss_backward(int num_levels, const b200_rpn_loss_level* levels_host, int activation, const float* grad_losses_dev,
                                    const float* divisor_dev, b200_stream_t stream);

/* Fast R-CNN: cls_score (R, C), bbox_pred / bbox_targets / inside / outside weights (R, B), B = 4 C' >= 4, labels (R,)
 * int32 or int64 (label_is_int64), R >= 1.
 * b200_fast_rcnn_loss_forward  losses_out (2,) = (loss_cls = mean over R of -log_softmax(cls_score)[label], loss_bbox = smooth L1
 *   with beta = 1 summed, / R); accuracy_out (1,) = mean of (argmax == label), argmax the first maximal index with NaN
 *   maximal.  A label outside [0, C) is never used as an index: loss_cls is NaN and the row counts as a miss.  One launch.
 * b200_fast_rcnn_loss_backward  cls_grad (R, C) = (softmax - onehot) * grad_losses[0] / R (a row with a label outside [0, C) is
 *   NaN) and bbox_grad (R, B) from grad_losses_dev (2,); either output may be null (not computed).  One launch. */
B200_API int b200_fast_rcnn_loss_forward(int num_rois, int num_classes, int bbox_width, const float* cls_score_dev, const float* bbox_pred_dev,
                                         const void* labels_dev, int label_is_int64, const float* bbox_targets_dev,
                                         const float* inside_weights_dev, const float* outside_weights_dev, void* workspace,
                                         size_t workspace_bytes, float* losses_out_dev, float* accuracy_out_dev, b200_stream_t stream);
B200_API int b200_fast_rcnn_loss_backward(int num_rois, int num_classes, int bbox_width, const float* cls_score_dev, const float* bbox_pred_dev,
                                          const void* labels_dev, int label_is_int64, const float* bbox_targets_dev,
                                          const float* inside_weights_dev, const float* outside_weights_dev, const float* grad_losses_dev,
                                          float* cls_grad_out_dev, float* bbox_grad_out_dev, b200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* B200_ROI_OPS_H_ */
