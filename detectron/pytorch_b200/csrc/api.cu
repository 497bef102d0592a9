// api.cu -- the library-wide entry points of libb200_roi_ops.so (version, status strings, launch count, options, debug buffers)
// and the RoIAlign forward / backward path dispatch (see include/b200_roi_ops.h).  Every other entry point is defined beside
// its kernels, in its op's translation unit.
#include "common.cuh"
#include <map>
#include <mutex>
#include <stdlib.h>
#include <string.h>
#include <utility>

namespace b200 {
unsigned long long g_launch_count = 0;

// Per-device kernel setup: the dynamic shared-memory limit recorded for each (kernel, device) pair and each device's SM
// count.  Both live in the device's context, so they are kept per device ordinal.
static std::mutex g_setup_mu;
static std::map<std::pair<const void*, int>, size_t> g_smem_limit;
static std::map<int, int> g_sm_count;

int smem_opt_in(const void* kernel, size_t bytes) {
    if (bytes <= 48 * 1024) return B200_ROI_OK;
    int dev = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err != cudaSuccess) { (void)cudaGetLastError(); return (int)err; }
    std::lock_guard<std::mutex> lock(g_setup_mu);
    size_t& limit = g_smem_limit[{kernel, dev}];
    if (limit >= bytes) return B200_ROI_OK;
    err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (err != cudaSuccess) { (void)cudaGetLastError(); return (int)err; }
    limit = bytes;
    return B200_ROI_OK;
}

int device_sm_count(int* sm_count) {
    int dev = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err != cudaSuccess) { (void)cudaGetLastError(); return (int)err; }
    std::lock_guard<std::mutex> lock(g_setup_mu);
    auto it = g_sm_count.find(dev);
    if (it == g_sm_count.end()) {
        int n = 0;
        err = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (err != cudaSuccess) { (void)cudaGetLastError(); return (int)err; }
        it = g_sm_count.emplace(dev, n).first;
    }
    *sm_count = it->second;
    return B200_ROI_OK;
}

static const char* const kOptionNames[kNumOptions] = {"B200_ROI_ALIGN_PATH", "B200_ROI_ALIGN_BWD_PATH"};
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

void b200_roi_ops_debug_timing_buffer(void* host_pinned) {
    roi_align_stream_set_debug_buffer((unsigned long long*)host_pinned);      // watchdog records of the streaming-strip path
    roi_align_strip_set_debug_buffer((unsigned long long*)host_pinned);       // watchdog records of the quad-strip path
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

}  // extern "C"
