// roi_align_tiled.cu -- Caffe2-exact RoIAlign FORWARD, feature-map-stationary ("tiled") fast path.
//
// Why: the RoI-centric gather (reference kernel, and our generic path) is bound by L1/L2
// transactions, not HBM: every 4-byte tap costs a 32-byte sector slot.  Here every feature byte
// crosses L2 -> SM once (+ a 1-cell halo): a work item = spatial tile x 32 channels is staged into
// shared memory TRANSPOSED to [cell][channel] (coalesced 128-byte row loads, conflict-free 128-bit
// shared stores) and then serves every bilinear SAMPLE whose top-left tap lies in the tile with
// conflict-free 128-bit shared loads: lane = (bin of a 4-bin group, 4-channel group), so one
// LDS.128 fetches one tap for 4 bins x 32 channels; the interpolation works on channel pairs (fma2, roi_align_tiled.cuh).
//
// Work assignment is per sample, not per bin: a sample's 4 taps span 2x2 cells, so a 1-cell halo is
// enough for ANY RoI size.  Bins whose samples fall into different tiles ("split" bins, ~1 in 5 at
// BASELINE cfg2) are finished with red.global.add of the partial means; the prepass zero-fills
// exactly those output elements.  Everything else is written once with plain stores, staged through
// shared memory so that the lanes of a store are consecutive bins of one channel.
//
// The prepass (one CTA per RoI) does everything that is channel independent exactly once: the
// per-axis sample tables (all IEEE divisions), and the list of RoIs per tile (global atomics), so the
// main kernel neither computes coordinates nor scans RoIs.  The main kernel is persistent (two CTAs
// per SM pulling (tile, channel group) items from a global counter), which removes the per-CTA launch
// cost and lets the two co-resident CTAs drift apart so one stages while the other computes.
//
// Numerics: each lane evaluates the reference's rounding recipe in the reference's order
// (oracle/roi_ops_oracle.c), so unsplit bins are bit-identical to the reference kernel; split bins
// differ by the association of <= 4 partial sums (~1 ulp).
//
// Semantics: lib/modeling/roi_xfrom/roi_align/src/roi_align_kernel.cu (reference) :16-63, :65-121.
#include "roi_align_tiled.cuh"
#include <stdlib.h>

namespace b200 {

// ------------------------------------------------------------------------------------------------
// prepass
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
roi_align_tiled_prep(const float* __restrict__ rois, float scale, int N, int R, int C, int H, int W, int PH, int PW, int sr,
                     int ny, int nx, int core_h, int core_w, int tiles_y, int tiles_x,
                     RoiHeader* __restrict__ hdr, AxisEntry* __restrict__ ytab, AxisEntry* __restrict__ xtab,
                     int* __restrict__ tile_count, unsigned* __restrict__ tile_list, int groups_max, float* __restrict__ out,
                     const int* __restrict__ row_map, int zero_split) {
    __shared__ int s_ty[kAxisMax], s_tx[kAxisMax];
    // the tile rows / cols that hold samples of this RoI (at most one per sample; the RoI's tile rectangle can span many
    // more), and the bin rows / cols the RoI has in each
    __shared__ int s_tile_y[kAxisMax], s_tile_x[kAxisMax];
    __shared__ int s_nbin_y[kAxisMax], s_nbin_x[kAxisMax];
    __shared__ int s_nty, s_ntx;
    __shared__ unsigned short s_split[kAxisMax * kAxisMax];
    __shared__ int s_nsplit;
    const int r = blockIdx.x;
    const XfromRoi g = xfrom_roi(rois + 5 * (size_t)r, scale, PH, PW, sr);
    const int t = threadIdx.x;
    if (t == 0) s_nsplit = 0;
    if (t < ny + nx) {
        const bool isy = t < ny;
        const int s = isy ? t : t - ny;
        const AxisEntry e = tiled_axis_entry(g, isy, s, sr, H, W);
        if (isy) { ytab[(size_t)r * ny + s] = e; s_ty[s] = e.low / core_h; }
        else     { xtab[(size_t)r * nx + s] = e; s_tx[s] = e.low / core_w; }
    }
    __syncthreads();
    const bool batch_ok = g.batch >= 0 && g.batch < N;
    // sample lows are monotone along an axis, so the tiles of this RoI form the rectangle below
    const int ty0 = s_ty[0], ty1 = s_ty[ny - 1], tx0 = s_tx[0], tx1 = s_tx[nx - 1];
    if (t == 0) {
        RoiHeader h;
        h.batch = batch_ok ? g.batch : -1;
        h.y_min = ty0; h.y_max = ty1; h.x_min = tx0; h.x_max = tx1;
        h.pad0 = h.pad1 = h.pad2 = 0;
        hdr[r] = h;
    }
    // Work entries: one per (tile, 8-bin group of this RoI in that tile), so that no warp of the main kernel is
    // ever stuck with more than 8 bins while its CTA waits.  The bin rectangle of a tile is derived exactly as
    // the main kernel derives it: [first sample in tile / sr, last sample in tile / sr] per axis.  Tiles without a
    // sample of the RoI get no entry; a tall or wide RoI can span more than kAxisMax tile rows / cols, but only the
    // (at most ny / nx) tiles that hold samples are listed, in ascending order.
    if (t < ny + nx) {
        const bool isy = t < ny;
        const int s = isy ? t : t - ny;
        const int* arr = isy ? s_ty : s_tx;
        const int cnt = isy ? ny : nx;
        if (s == 0 || arr[s] != arr[s - 1]) {                 // first sample of its tile (lows are monotone along an axis)
            int rank = 0;
            for (int j = 1; j <= s; ++j) rank += arr[j] != arr[j - 1];
            int last = s;
            while (last + 1 < cnt && arr[last + 1] == arr[s]) ++last;
            const int nbin = last / sr - s / sr + 1;
            if (isy) { s_tile_y[rank] = arr[s]; s_nbin_y[rank] = nbin; } else { s_tile_x[rank] = arr[s]; s_nbin_x[rank] = nbin; }
            if (last == cnt - 1) { if (isy) s_nty = rank + 1; else s_ntx = rank + 1; }
        }
    }
    __syncthreads();
    const int nty = s_nty, ntx = s_ntx;
    if (batch_ok) {
        for (int k = t; k < nty * ntx; k += blockDim.x) {
            const int ky = k / ntx, kx = k - ky * ntx;
            const int nb = s_nbin_y[ky] * s_nbin_x[kx];
            const int ngroups = (nb + kStageBins - 1) / kStageBins;
            const int tile = (g.batch * tiles_y + s_tile_y[ky]) * tiles_x + s_tile_x[kx];
            const int pos = atomicAdd(&tile_count[tile], ngroups);
            unsigned* dst = tile_list + (size_t)tile * R * groups_max + pos;
            for (int gI = 0; gI < ngroups; ++gI) dst[gI] = (unsigned)r | ((unsigned)gI << 16);
        }
    }
    // bins the main kernel accumulates into (their samples straddle tiles) or never visits (bad batch index)
    if (!zero_split) return;                         // the host zero-filled the whole output instead
    const int bins = PH * PW;
    for (int bin = t; bin < bins; bin += blockDim.x) {
        const int ph = bin / PW, pw = bin % PW;
        bool split = !batch_ok;
        for (int i = 1; i < sr; ++i) split |= (s_ty[ph * sr + i] != s_ty[ph * sr]) || (s_tx[pw * sr + i] != s_tx[pw * sr]);
        if (split) s_split[atomicAdd(&s_nsplit, 1)] = (unsigned short)bin;
    }
    __syncthreads();
    const int nsplit = s_nsplit;
    float* out_r = out + (size_t)(row_map ? row_map[r] : r) * C * bins;
    for (int idx = t; idx < C * nsplit; idx += blockDim.x) {
        const int c = idx / nsplit, k = idx - c * nsplit;
        out_r[(size_t)c * bins + s_split[k]] = 0.f;
    }
}

// ------------------------------------------------------------------------------------------------
// main kernel (persistent)
// ------------------------------------------------------------------------------------------------
template <int SR>
__global__ void __launch_bounds__(kTiledThreads, kTiledCtasPerSM)
roi_align_tiled_fwd(const float* __restrict__ bottom, const AxisEntry* __restrict__ g_ytab, const AxisEntry* __restrict__ g_xtab,
                    int* __restrict__ work_counter, const int* __restrict__ tile_count,
                    const unsigned* __restrict__ tile_list, int list_stride, float* __restrict__ out,
                    int N, int R, int C, int H, int W, int PH, int PW, int ny, int nx,
                    int core_h, int core_w, int tile_h, int tiles_y, int tiles_x, int n_cgroups, int n_work,
                    const int* __restrict__ row_map) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* tile = reinterpret_cast<float*>(smem_raw);
    AxisEntry* wtab_all = reinterpret_cast<AxisEntry*>(smem_raw + (size_t)kTX * tile_h * kCellWords * 4);
    float* stage_all = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(wtab_all) + (size_t)kWarps * (ny + nx) * 16);
    int* misc = reinterpret_cast<int*>(stage_all + kWarps * kCG * kStageWords);   // [0]=work item, [1]=next RoI of the list

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int bins = PH * PW;
    constexpr float kCount = (float)(SR * SR);
    constexpr unsigned kFull = (1u << SR) - 1u;
    AxisEntry* wy = wtab_all + warp * (ny + nx);
    AxisEntry* wx = wy + ny;
    float* stage = stage_all + warp * kCG * kStageWords;
    const int q = lane >> 3, i = lane & 7;                // compute mapping: (bin of the 4-bin group, 4-channel group)
    const int cs = lane >> 3, bb = lane & 7;              // flush mapping:   (channel within a group of 4, staged bin)
    const size_t plane = (size_t)H * W;

    if (tid == 0) misc[0] = atomicAdd(work_counter, 1);
    for (;;) {
        __syncthreads();                                  // misc[0] published; previous item fully consumed
        const int work = misc[0];
        if (work >= n_work) break;
        // the NEXT item is claimed now, so the global atomic's latency hides behind this item
        int next_work = 0;
        if (tid == 0) { next_work = atomicAdd(work_counter, 1); misc[1] = 0; }
        const int tile_id = work / n_cgroups;             // consecutive items share a tile (same list, tables hit L2)
        const int c0 = (work - tile_id * n_cgroups) * kCG;
        const int n_list = tile_count[tile_id];
        if (n_list == 0) {                                // uniform: nothing samples this tile
            __syncthreads();
            if (tid == 0) misc[0] = next_work;
            continue;
        }
        const unsigned* list = tile_list + (size_t)tile_id * list_stride;
        const int tx = tile_id % tiles_x, ty = (tile_id / tiles_x) % tiles_y, n = tile_id / (tiles_x * tiles_y);
        const int y0 = ty * core_h, x0 = tx * core_w;
        const int y_end = y0 + core_h, x_end = x0 + core_w;      // core = [y0, y_end) x [x0, x_end)

        // ---- stage the tile: rows [y0, y0+tile_h) x cols [x0, x0+32) x channels [c0, c0+32), zero outside the map.
        // Loads are branch-free (addresses clamped into the tensor, invalid lanes zeroed afterwards) and issued
        // kRowsPerBatch rows = 4*kRowsPerBatch independent 128-byte-coalesced loads at a time (20 per thread,
        // x 1024 resident threads per SM in flight).
        {
            // 16 warps: warp w stages channel quad (w & 7) of the rows of parity (w >> 3)
            constexpr int kRowsPerBatch = 5;
            const int x = x0 + lane;
            const bool x_ok = x < W;
            const int cq = c0 + 4 * (warp & 7);
            const bool ch0 = cq < C, ch1 = cq + 1 < C, ch2 = cq + 2 < C, ch3 = cq + 3 < C;
            const float* base = bottom + (size_t)n * C * plane + min(x, W - 1);
            const float* p0 = base + (size_t)min(cq, C - 1) * plane;
            const float* p1 = base + (size_t)min(cq + 1, C - 1) * plane;
            const float* p2 = base + (size_t)min(cq + 2, C - 1) * plane;
            const float* p3 = base + (size_t)min(cq + 3, C - 1) * plane;
            float* dst = tile + (size_t)lane * kCellWords + 4 * (warp & 7);
            constexpr int kPar = kWarps / 8;              // row parities staged concurrently
            for (int k0 = (warp >> 3); k0 < tile_h; k0 += kPar * kRowsPerBatch) {
                float4 v[kRowsPerBatch];
#pragma unroll
                for (int bq = 0; bq < kRowsPerBatch; ++bq) {
                    const size_t off = (size_t)min(y0 + k0 + kPar * bq, H - 1) * W;
                    v[bq].x = __ldg(p0 + off); v[bq].y = __ldg(p1 + off); v[bq].z = __ldg(p2 + off); v[bq].w = __ldg(p3 + off);
                }
#pragma unroll
                for (int bq = 0; bq < kRowsPerBatch; ++bq) {
                    const int row = k0 + kPar * bq;
                    if (row < tile_h) {
                        const bool ok = x_ok && (y0 + row < H);
                        float4 o;
                        o.x = (ok && ch0) ? v[bq].x : 0.f; o.y = (ok && ch1) ? v[bq].y : 0.f;
                        o.z = (ok && ch2) ? v[bq].z : 0.f; o.w = (ok && ch3) ? v[bq].w : 0.f;
                        *reinterpret_cast<float4*>(dst + (size_t)row * kTX * kCellWords) = o;
                    }
                }
            }
        }
        __syncthreads();

        // ---- warps pull RoIs of this tile; the axis tables of the NEXT RoI are fetched into registers
        //      while the current one is processed
        int item = 0;
        if (lane == 0) item = atomicAdd(&misc[1], 1);
        item = __shfl_sync(0xffffffffu, item, 0);
        AxisEntry pre_y, pre_x;
        pre_y.low = pre_x.low = 0; pre_y.valid = pre_x.valid = 0; pre_y.l = pre_y.h = pre_x.l = pre_x.h = 0.f;
        unsigned entry = 0;
        if (item < n_list) {
            entry = list[item];
            const int r = entry & 0xffffu;
            if (lane < ny) pre_y = g_ytab[(size_t)r * ny + lane];
            if (lane < nx) pre_x = g_xtab[(size_t)r * nx + lane];
        }
        while (item < n_list) {
            // Tile-local tables of this RoI: every lane converts its own axis sample into
            // {shared-memory offset of the low cell (words), weight of the high cell, weight of the low cell};
            // samples that are not this tile's (low cell outside the core) or that the reference skips (outside
            // the map) get offset 0 and zero weights, so the inner loop needs no checks: they contribute +0.
            bool in_y = false, in_x = false;
            AxisEntry ty_e, tx_e;
            ty_e.low = 0; ty_e.valid = 0; ty_e.l = 0.f; ty_e.h = 0.f;
            tx_e = ty_e;
            if (lane < ny) {
                in_y = pre_y.low >= y0 && pre_y.low < y_end;
                if (in_y && pre_y.valid) { ty_e.low = (pre_y.low - y0) * (kTX * kCellWords); ty_e.l = pre_y.l; ty_e.h = pre_y.h; }
            }
            if (lane < nx) {
                in_x = pre_x.low >= x0 && pre_x.low < x_end;
                if (in_x && pre_x.valid) { tx_e.low = (pre_x.low - x0) * kCellWords; tx_e.l = pre_x.l; tx_e.h = pre_x.h; }
            }
            __syncwarp();
            if (lane < ny) wy[lane] = ty_e;
            if (lane < nx) wx[lane] = tx_e;
            __syncwarp();
            const int r_cur = entry & 0xffffu, kb = (int)(entry >> 16) * kStageBins;
            if (lane == 0) item = atomicAdd(&misc[1], 1);
            item = __shfl_sync(0xffffffffu, item, 0);
            if (item < n_list) {
                entry = list[item];
                const int r = entry & 0xffffu;
                if (lane < ny) pre_y = g_ytab[(size_t)r * ny + lane];
                if (lane < nx) pre_x = g_xtab[(size_t)r * nx + lane];
            }
            // samples of this RoI whose low cell lies in this tile's core: contiguous index ranges (bit masks)
            const unsigned my = __ballot_sync(0xffffffffu, in_y), mx = __ballot_sync(0xffffffffu, in_x);
            if (my == 0u || mx == 0u) continue;
            const int ph0 = (__ffs(my) - 1) / SR, ph1 = (31 - __clz(my)) / SR + 1;
            const int pw0 = (__ffs(mx) - 1) / SR, pw1 = (31 - __clz(mx)) / SR + 1;
            const int npw = pw1 - pw0, nb = (ph1 - ph0) * npw;
            const unsigned div_m = 65536u / (unsigned)npw + 1u;          // b / npw == (b * div_m) >> 16 for b < 1024
            float* out_r = out + (size_t)(row_map ? row_map[r_cur] : r_cur) * C * bins + (size_t)c0 * bins;
            const float* tbase = tile + 4 * i;
            if (kb < nb) {                                   // always true for entries the prepass wrote
#pragma unroll
                for (int jj = 0; jj < kStageBins / 4; ++jj) {
                    const int b = kb + jj * 4 + q;
                    const int bc = min(b, nb - 1);                   // lanes past the end recompute the last bin, unstored
                    const int dph = (int)(((unsigned)bc * div_m) >> 16);
                    const int sy = (ph0 + dph) * SR, sx = (pw0 + (bc - dph * npw)) * SR;
                    u64x acc_lo = 0ull, acc_hi = 0ull;               // channels (0,1) and (2,3) of this lane's group
#pragma unroll
                    for (int iy = 0; iy < SR; ++iy) {
                        const AxisEntry ey = wy[sy + iy];
#pragma unroll
                        for (int ix = 0; ix < SR; ++ix) {
                            const AxisEntry ex = wx[sx + ix];
                            const float w1 = __fmul_rn(ey.h, ex.h), w2 = __fmul_rn(ey.h, ex.l);
                            const float w3 = __fmul_rn(ey.l, ex.h), w4 = __fmul_rn(ey.l, ex.l);
                            const u64x W1 = pack2(w1, w1), W2 = pack2(w2, w2), W3 = pack2(w3, w3), W4 = pack2(w4, w4);
                            const float* p = tbase + (ey.low + ex.low);
                            const ulonglong2 v1 = lds128(p), v2 = lds128(p + kCellWords);
                            const ulonglong2 v3 = lds128(p + kTX * kCellWords), v4 = lds128(p + (kTX + 1) * kCellWords);
                            // val = FFMA(v4,w4, FFMA(v3,w3, FFMA(v1,w1, FMUL(v2,w2))));  acc += val   (reference order)
                            acc_lo = add2(acc_lo, fma2(v4.x, W4, fma2(v3.x, W3, fma2(v1.x, W1, mul2(v2.x, W2)))));
                            acc_hi = add2(acc_hi, fma2(v4.y, W4, fma2(v3.y, W3, fma2(v1.y, W1, mul2(v2.y, W2)))));
                        }
                    }
                    float a0, a1, a2, a3;
                    unpack2(acc_lo, a0, a1); unpack2(acc_hi, a2, a3);
                    if (SR == 3) {        // count 9: a true division, like the reference's `output_val /= count`
                        a0 = __fdiv_rn(a0, kCount); a1 = __fdiv_rn(a1, kCount); a2 = __fdiv_rn(a2, kCount); a3 = __fdiv_rn(a3, kCount);
                    } else {              // count 1 / 4 / 16: multiplying by the reciprocal is exact
                        a0 = __fmul_rn(a0, 1.f / kCount); a1 = __fmul_rn(a1, 1.f / kCount);
                        a2 = __fmul_rn(a2, 1.f / kCount); a3 = __fmul_rn(a3, 1.f / kCount);
                    }
                    if (b < nb) {
                        float* st = stage + (4 * i) * kStageWords + jj * 4 + q;       // [channel][bin]
                        st[0] = a0; st[kStageWords] = a1; st[2 * kStageWords] = a2; st[3 * kStageWords] = a3;
                    }
                }
                __syncwarp();
                // -- flush 8 bins x 32 channels: lanes = (channel within a group of 4, bin)
                const int b = kb + bb;
                if (b < nb) {
                    const int dph = (int)(((unsigned)b * div_m) >> 16);
                    const int ph = ph0 + dph, pw = pw0 + (b - dph * npw);
                    const bool whole = (((my >> (ph * SR)) & kFull) == kFull) && (((mx >> (pw * SR)) & kFull) == kFull);
                    float* dst = out_r + ph * PW + pw + (size_t)cs * bins;
                    const float* src = stage + cs * kStageWords + bb;
                    const int cmax = C - c0 - cs;                   // channel c = 4*cb + cs is real iff 4*cb < cmax
                    if (whole) {
#pragma unroll
                        for (int cb = 0; cb < kCG / 4; ++cb)
                            if (4 * cb < cmax) dst[(size_t)(4 * cb) * bins] = src[4 * cb * kStageWords];
                    } else {
#pragma unroll
                        for (int cb = 0; cb < kCG / 4; ++cb)
                            if (4 * cb < cmax) atomicAdd(dst + (size_t)(4 * cb) * bins, src[4 * cb * kStageWords]);
                    }
                }
                __syncwarp();
            }
        }
        __syncthreads();                                  // every warp has read misc[0] and is done with the tile
        if (tid == 0) misc[0] = next_work;
    }
}

size_t roi_align_tiled_workspace_bytes(int N, int R, int H, int W, int PH, int PW, int sr) {
    TiledPlan p;
    if (!roi_align_tiled_plan(N, R, H, W, 1, PH, PW, sr, &p)) return 0;
    return p.ws_bytes;
}

// returns B200_ROI_OK when the fast path ran; kPathDeclined when it does not apply (caller falls back)
int roi_align_forward_tiled(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                            const float* rois, float* top, const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    TiledPlan p;
    if (!roi_align_tiled_plan(N, R, H, W, C, PH, PW, sr, &p)) return kPathDeclined;
    if (workspace == nullptr || workspace_bytes < p.ws_bytes) return kPathDeclined;
    unsigned char* ws = (unsigned char*)workspace;
    RoiHeader* hdr = (RoiHeader*)(ws + p.hdr_off);
    AxisEntry* ytab = (AxisEntry*)(ws + p.ytab_off);
    AxisEntry* xtab = (AxisEntry*)(ws + p.xtab_off);
    int* zero = (int*)(ws + p.zero_off);
    int* work_counter = zero;
    int* tile_count = zero + 4;
    unsigned* tile_list = (unsigned*)(ws + p.tile_list_off);

    const auto fwd = sr == 1 ? roi_align_tiled_fwd<1> : sr == 2 ? roi_align_tiled_fwd<2> : sr == 3 ? roi_align_tiled_fwd<3> : roi_align_tiled_fwd<4>;
    int sms = 0;
    int rc = smem_opt_in(fwd, (228 * 1024 - kTiledCtasPerSM * 1024) / kTiledCtasPerSM);
    if (rc == B200_ROI_OK) rc = device_sm_count(&sms);
    if (rc != B200_ROI_OK) return rc;
    cudaError_t err = cudaMemsetAsync(zero, 0, p.zero_bytes, stream);
    if (err != cudaSuccess) return (int)err;
    // The bins the main kernel accumulates into must start at zero.  With a dense output one memset of the whole tensor
    // (25.7 MB at cfg2) is cheaper than the prepass storing ~1.3 M scattered zeros; the indexed variant shares
    // its output tensor with other calls and zero-fills exactly its own split bins.
    const bool whole = row_map == nullptr;
    if (whole) {
        err = cudaMemsetAsync(top, 0, sizeof(float) * (size_t)R * C * PH * PW, stream);
        if (err != cudaSuccess) return (int)err;
    }
    roi_align_tiled_prep<<<R, 128, 0, stream>>>(rois, scale, N, R, C, H, W, PH, PW, sr, p.ny, p.nx, p.core_h, p.core_w,
                                               p.tiles_y, p.tiles_x, hdr, ytab, xtab, tile_count, tile_list, p.groups_max, top, row_map,
                                               whole ? 0 : 1);
    const int n_cgroups = (C + kCG - 1) / kCG;
    const int n_work = p.tiles_total * n_cgroups;
    const int grid = n_work < kTiledCtasPerSM * sms ? n_work : kTiledCtasPerSM * sms;      // persistent CTAs
    fwd<<<grid, kTiledThreads, p.smem_bytes, stream>>>(bottom, ytab, xtab, work_counter, tile_count, tile_list, R * p.groups_max, top,
                                                       N, R, C, H, W, PH, PW, p.ny, p.nx, p.core_h, p.core_w, p.tile_h, p.tiles_y,
                                                       p.tiles_x, n_cgroups, n_work, row_map);
    return finish_launch(2);
}

}  // namespace b200
