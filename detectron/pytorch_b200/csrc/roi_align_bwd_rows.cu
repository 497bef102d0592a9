// roi_align_bwd_rows.cu -- Caffe2-exact RoIAlign BACKWARD, row-stationary gather path (no global atomics).
//
// The scatter formulations (reference kernel, our generic and NHWC paths) are bound by the L2 atomic unit: one
// reduction per tap (per 4 channels at best), plus a zero-fill of dX (and a transpose for the NHWC variant).  Here
// the roles are swapped: a work item is one image ROW of one 32-cell x-tile for one block of 64 / 128 channels; ONE
// WARP owns the item's accumulator ([cell][channel] in shared memory, lane = 2 / 4 adjacent channels), visits every
// bilinear tap that lands in it and read-modify-writes the accumulator with plain 64/128-bit shared accesses.  Each
// dX element is produced by exactly one warp and written exactly once with coalesced 128-byte stores, so there is
// no memset of dX, no floating-point atomic and no scratch image; accumulation inside an item is sequential.
//
//   tables (1 launch, parallel)  per-RoI axis sample tables (all IEEE divisions) and, in the same launch,
//                                dY (R, C, PH, PW) -> dYt (R, PH, PW, C) / count: channel-innermost, so that a
//                                warp reads the gradient of a bin for its channels with one coalesced access.
//                                Every valid y-sample of every RoI contributes two "units" (row of its low cell
//                                with weight hy, row of its high cell with weight ly); the table threads append
//                                them to fixed-capacity per-row lists (one atomicAdd on the row's counter each;
//                                units beyond the capacity go to one overflow list that every row scans --
//                                correct for any input, fast for all but pathological RoI pile-ups).
//   main   (persistent warps)    item <- atomic counter; zero accumulator; for each unit of the row whose RoI
//                                overlaps the x-tile: lanes j < PW*sr build the tap records of x-sample j (cell
//                                offset, wy * wx), staged in shared memory; the gradients of the needed bins are
//                                loaded to registers (software pipelined one unit ahead); taps are applied with
//                                LDS / FFMA / STS (taps outside the tile land in a scratch cell instead of
//                                being branched around).  Finally the row segment is transposed to NCHW on the
//                                way out.
//
// Numerics: per tap the term is (dY / count) * (wy * wx) with count = sr^2 in {1, 4}: the division is an exact
// scaling, so each addend equals the reference's FMUL(dY, w) / count up to the fused multiply-add's single rounding (the
// product is not rounded separately inside fma2); the order of the additions differs as well, as it does between two runs of
// the reference's atomicAdd.  Against the fp64 oracle it is no further off than the reference kernel itself
// (test_backward_tolerance_is_derived_from_the_reference_kernels_own_spread, tests/golden/roi_align_bwd_spread.npz).
//
// Semantics: lib/modeling/roi_xfrom/roi_align/src/roi_align_kernel.cu (reference) :150-193, :195-270.
#include "roi_align_tiled.cuh"
#include <stdlib.h>

namespace b200 {

constexpr int kRowCells = 32;             // cells per x-tile = lanes of the write-out
constexpr int kTableThreads = 256;
constexpr int kTransposeChannelsMax = 256; // channels per transpose CTA (whole 1 KB rows of the channel-innermost copy at C = 256)
constexpr int kRankRows = 1024;           // N * H up to which the main kernel orders the rows by weight

struct __align__(16) BwdRoi {
    int batch;                            // -1: batch index out of range (contributes nothing)
    int x_lo, x_hi;                       // range of cells any x-sample of the RoI can touch
    int y_lo, y_hi;                       // same for rows
    int pad0, pad1, pad2;
};

__device__ __forceinline__ unsigned smem_u32addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ AxisEntry make_axis_zero() { AxisEntry e; e.low = 0; e.valid = 0; e.l = 0.f; e.h = 0.f; return e; }

struct RowsPlan {
    int ny, nx, tiles_x, rows, row_cap;
    size_t roi_off, xtab_off, zero_off, zero_bytes, row_list_off, ovf_off, dyt_off, ws_bytes;
};

static bool rows_plan(int N, int R, int C, int H, int W, int PH, int PW, int sr, RowsPlan* p) {
    if (sr < 1 || sr > 2 || (PW != 7 && PW != 14) || PH * sr > kAxisMax || PW * sr > kAxisMax) return false;
    if (R <= 0 || R > 65535 || N <= 0 || C <= 0 || (C % 64) != 0 || H <= 0 || W <= 0) return false;
    if (H > 65535) return false;
    if ((long long)R * C * PH * PW >= (1LL << 31) || (long long)N * C * H * W >= (1LL << 31)) return false;
    p->ny = PH * sr; p->nx = PW * sr; p->tiles_x = (W + kRowCells - 1) / kRowCells; p->rows = N * H;
    size_t off = 0;
    p->roi_off = off;      off = align_up(off + (size_t)R * sizeof(BwdRoi), 256);
    p->xtab_off = off;     off = align_up(off + (size_t)R * p->nx * sizeof(AxisEntry), 256);
    // zeroed per call: [0] item counter, [1] overflow count, [4 ..] units per row
    p->zero_off = off;     p->zero_bytes = align_up(((size_t)p->rows + 4) * sizeof(int), 256); off += p->zero_bytes;
    const long long total_units = 2LL * R * p->ny;
    long long cap = 8 * ((total_units + p->rows - 1) / p->rows);            // 8x the mean row population
    if (cap < 64) cap = 64;
    if (cap > total_units) cap = total_units;
    if (cap * p->rows * 8 > (64LL << 20)) cap = (64LL << 20) / (8LL * p->rows);
    if (cap < 32) return false;
    p->row_cap = (int)cap;
    p->row_list_off = off; off = align_up(off + (size_t)p->rows * p->row_cap * sizeof(uint2), 256);
    p->ovf_off = off;      off = align_up(off + (size_t)total_units * sizeof(uint4), 256);
    p->dyt_off = off;      off = align_up(off + (size_t)R * PH * PW * C * sizeof(float), 256);
    p->ws_bytes = off;
    return true;
}

// ------------------------------------------------------------------------------------------------
// tables + transpose (parallel)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTableThreads)
roi_align_bwd_rows_tables(const float* __restrict__ rois, const float* __restrict__ dy, float scale, int N, int R, int C, int H,
                          int W, int PH, int PW, int sr, int table_ctas, int tr_ch, BwdRoi* __restrict__ roi_out,
                          AxisEntry* __restrict__ xtab, int* __restrict__ zeroed, uint2* __restrict__ row_list, int row_cap,
                          uint4* __restrict__ ovf, float* __restrict__ dyt, const int* __restrict__ row_map) {
    extern __shared__ __align__(16) float s_tr[];
    const int tid = threadIdx.x;
    const int ny = PH * sr, nx = PW * sr;
    if ((int)blockIdx.x < table_ctas) {
        const int per = ny + nx;
        const int k = blockIdx.x * kTableThreads + tid;
        if (k >= R * per) return;
        const int r = k / per, s = k - r * per;
        const XfromRoi g = xfrom_roi(rois + 5 * (size_t)r, scale, PH, PW, sr);
        const bool isy = s < ny;
        const AxisEntry e = tiled_axis_entry(g, isy, isy ? s : s - ny, sr, H, W);
        if (isy) {                                                              // lows are monotone along an axis
            const bool batch_ok = g.batch >= 0 && g.batch < N;
            if (s == 0) { roi_out[r].batch = batch_ok ? g.batch : -1; roi_out[r].y_lo = e.low; }
            if (s == ny - 1) roi_out[r].y_hi = min(e.low + 1, H - 1);
            if (batch_ok && e.valid) {
                const unsigned key = (unsigned)r | ((unsigned)s << 16);
#pragma unroll
                for (int which = 0; which < 2; ++which) {                       // row of the low cell: hy; of the high cell: ly
                    const int row = g.batch * H + (which ? min(e.low + 1, H - 1) : e.low);
                    const uint2 u = make_uint2(key | (which ? 0x80000000u : 0u), __float_as_uint(which ? e.l : e.h));
                    const int pos = atomicAdd(&zeroed[4 + row], 1);
                    if (pos < row_cap) row_list[(size_t)row * row_cap + pos] = u;
                    else ovf[atomicAdd(&zeroed[1], 1)] = make_uint4(u.x, u.y, (unsigned)row, 0u);
                }
            }
        } else {
            xtab[(size_t)r * nx + (s - ny)] = e;
            if (s == ny) roi_out[r].x_lo = e.low;
            if (s == per - 1) roi_out[r].x_hi = min(e.low + 1, W - 1);
        }
        return;
    }
    // ---- dY (r, c, bin) -> dYt (r, bin, c) / count for one RoI and one block of channels
    const int bins = PH * PW;
    const int cblocks = (C + tr_ch - 1) / tr_ch;
    const int t = blockIdx.x - table_ctas;
    const int r = t / cblocks, c0 = (t - r * cblocks) * tr_ch;
    const int cc = min(tr_ch, C - c0);
    const int stride = bins | 1;                            // odd: the transposed read below is bank-conflict free
    const int lane = tid & 31, warp = tid >> 5;
    constexpr int kWarps = kTableThreads / 32;
    const float* src = dy + ((size_t)(row_map ? row_map[r] : r) * C + c0) * bins;
    const float inv = 1.f / (float)(sr * sr);               // count in {1, 4}: multiplying by the reciprocal is the exact division
    if (stride == bins && ((cc * bins) & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        // odd bin count: the block is copied linearly, 16 bytes at a time
        const float4* src4 = reinterpret_cast<const float4*>(src);
        float4* s4 = reinterpret_cast<float4*>(s_tr);
        for (int k = tid; k < (cc * bins) >> 2; k += kTableThreads) {
            float4 v = __ldg(src4 + k);
            v.x = __fmul_rn(v.x, inv); v.y = __fmul_rn(v.y, inv); v.z = __fmul_rn(v.z, inv); v.w = __fmul_rn(v.w, inv);
            s4[k] = v;
        }
    } else if (stride == bins) {
        for (int k = tid; k < cc * bins; k += kTableThreads) s_tr[k] = __fmul_rn(src[k], inv);
    } else {
        for (int c = warp; c < cc; c += kWarps)
            for (int b = lane; b < bins; b += 32) s_tr[c * stride + b] = __fmul_rn(src[c * bins + b], inv);
    }
    __syncthreads();
    float* dst = dyt + (size_t)r * bins * C + c0;
    for (int b = warp; b < bins; b += kWarps)
        for (int c = lane; c < cc; c += 32) dst[(size_t)b * C + c] = s_tr[c * stride + b];
}

// ------------------------------------------------------------------------------------------------
// main kernel
// ------------------------------------------------------------------------------------------------
// Shared memory is addressed with 32-bit shared-window addresses and explicit ld/st.shared (volatile asm keeps the
// program order of the read-modify-writes, which may alias).
template <int CPL> struct Acc;
template <> struct Acc<2> {
    static constexpr int kHalves = 1;
    static __device__ __forceinline__ void ld(unsigned a, u64x (&v)[1]) { asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v[0]) : "r"(a)); }
    static __device__ __forceinline__ void st(unsigned a, const u64x (&v)[1]) { asm volatile("st.shared.b64 [%0], %1;" ::"r"(a), "l"(v[0]) : "memory"); }
    static __device__ __forceinline__ void ldg(const float* p, u64x (&v)[1]) { v[0] = __ldg(reinterpret_cast<const u64x*>(p)); }
};
template <> struct Acc<4> {
    static constexpr int kHalves = 2;
    static __device__ __forceinline__ void ld(unsigned a, u64x (&v)[2]) { asm volatile("ld.shared.v2.b64 {%0, %1}, [%2];" : "=l"(v[0]), "=l"(v[1]) : "r"(a)); }
    static __device__ __forceinline__ void st(unsigned a, const u64x (&v)[2]) { asm volatile("st.shared.v2.b64 [%0], {%1, %2};" ::"r"(a), "l"(v[0]), "l"(v[1]) : "memory"); }
    static __device__ __forceinline__ void ldg(const float* p, u64x (&v)[2]) { const ulonglong2 t = __ldg(reinterpret_cast<const ulonglong2*>(p)); v[0] = t.x; v[1] = t.y; }
};

template <int CPL> __host__ __device__ constexpr int rows_acc_stride() { return 33 * CPL; }          // words per cell (odd multiple of CPL)
template <int NX> __host__ __device__ constexpr int rows_stage_bytes() { return ((NX * 16 + 127) / 128) * 128; }
template <int CPL> __host__ __device__ constexpr int rows_acc_bytes() {                              // 32 cells + 1 scratch cell, 16-byte multiple
    return (((kRowCells + 1) * rows_acc_stride<CPL>() * 4 + 15) / 16) * 16;
}
template <int CPL, int NX> __host__ __device__ constexpr int rows_warp_smem() { return rows_acc_bytes<CPL>() + 2 * rows_stage_bytes<NX>(); }

template <int PW, int SR, int CPL, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, (CPL == 2 && PW == 7) ? 2 : 1)     // PW = 14: ~117 KB per CTA, a second CTA never fits (ADVICE r1)
roi_align_bwd_rows(const BwdRoi* __restrict__ roi_in, const AxisEntry* __restrict__ xtab, int* __restrict__ zeroed,
                   const uint2* __restrict__ row_list, int row_cap, const uint4* __restrict__ ovf, const float* __restrict__ dyt,
                   float* __restrict__ dx, int N, int C, int H, int W, int PH, int tiles_x) {
    constexpr int NX = PW * SR;
    constexpr int S = rows_acc_stride<CPL>();
    constexpr int CHB = 32 * CPL;                       // channels per item
    constexpr int HV = Acc<CPL>::kHalves;
    constexpr int SB = rows_stage_bytes<NX>();
    constexpr int kCellBytes = S * 4;
    constexpr int kTrash = kRowCells * kCellBytes;      // scratch cell: taps that fall outside the x-tile
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned acc_s = smem_u32addr(smem_raw) + (unsigned)warp * rows_warp_smem<CPL, NX>();
    const unsigned stage_s = acc_s + rows_acc_bytes<CPL>();
    const unsigned lane_acc = acc_s + lane * (CPL * 4);
    const int cblocks = C / CHB;
    const int items_per_row = tiles_x * cblocks;
    const int total = N * H * items_per_row;

    // Rows are handed out heaviest first (fewer stragglers at the end): every CTA derives the same order from the
    // per-row unit counts with a counting sort in shared memory (the accumulators are not in use yet).
    __shared__ unsigned short s_order[kRankRows];
    const int rows = N * H;
    const bool ranked = rows <= kRankRows;
    if (ranked) {
        int* hist = reinterpret_cast<int*>(smem_raw);               // [1024] bins by descending (clamped) count
        for (int k = threadIdx.x; k < 1024; k += WARPS * 32) hist[k] = 0;
        __syncthreads();
        for (int k = threadIdx.x; k < rows; k += WARPS * 32) atomicAdd(&hist[1023 - min(zeroed[4 + k], 1023)], 1);
        __syncthreads();
        if (warp == 0) {                                            // exclusive prefix, 32 bins per lane
            int sum = 0;
            for (int k = 0; k < 32; ++k) sum += hist[lane * 32 + k];
            int incl = sum;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
            int run = incl - sum;
            for (int k = 0; k < 32; ++k) { const int c = hist[lane * 32 + k]; hist[lane * 32 + k] = run; run += c; }
        }
        __syncthreads();
        // stable placement by one warp (the order must be the same in every CTA): rows in index order, 32 at a time
        if (warp == 0) {
            for (int base = 0; base < rows; base += 32) {
                const int k = base + lane;
                const bool valid = k < rows;
                const int b = valid ? 1023 - min(zeroed[4 + k], 1023) : 1024 + lane;
                const unsigned peers = __match_any_sync(0xffffffffu, b);
                const int start = valid ? hist[b] : 0;
                __syncwarp();
                if (valid && (peers & ((1u << lane) - 1u)) == 0u) hist[b] = start + __popc(peers);
                __syncwarp();
                if (valid) s_order[start + __popc(peers & ((1u << lane) - 1u))] = (unsigned short)k;
            }
        }
        __syncthreads();
    }

    for (;;) {
        int item = 0;
        if (lane == 0) item = atomicAdd(&zeroed[0], 1);
        item = __shfl_sync(0xffffffffu, item, 0);
        if (item >= total) break;
        const int slot = item / items_per_row;
        const int row = ranked ? (int)s_order[slot] : slot;
        const int rem = item - slot * items_per_row;
        const int cb = rem / tiles_x, tx = rem - cb * tiles_x;
        const int n = row / H, y = row - n * H;
        const int x0 = tx * kRowCells;
        const unsigned lane_ch = (unsigned)(cb * CHB + lane * CPL);     // all dYt offsets fit 32 bits (plan: R*C*PH*PW < 2^31)

        {   // zero the 32 cells of the accumulator: 32 * 33 lane-vectors
            u64x z[HV];
#pragma unroll
            for (int q = 0; q < HV; ++q) z[q] = 0ULL;
#pragma unroll 3
            for (int k = 0; k < 33; ++k) Acc<CPL>::st(lane_acc + k * (32 * CPL * 4), z);
        }
        __syncwarp();

        // A: tap records of x-sample `lane` of one unit into stage buffer `slot`, gradient loads of the bins it needs
        auto stage_a = [&](unsigned key, float wy, const AxisEntry& e, int slot, u64x (&G)[PW][HV]) -> unsigned {
            int off_lo = kTrash, off_hi = kTrash;
            float w_lo = 0.f, w_hi = 0.f;
            bool any = false;
            if (lane < NX && e.valid) {
                const int lo = e.low - x0, hi = min(e.low + 1, W - 1) - x0;
                if ((unsigned)lo < (unsigned)kRowCells) { off_lo = lo * kCellBytes; any = true; }
                // clamped at the last column (hi == lo): the high tap's weight is exactly 0 (xfrom_axis), drop it
                if ((unsigned)hi < (unsigned)kRowCells && hi != lo) { off_hi = hi * kCellBytes; any = true; }
                w_lo = __fmul_rn(wy, e.h);
                w_hi = __fmul_rn(wy, e.l);
            }
            if (lane < NX)
                asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(stage_s + slot * SB + lane * 16), "r"(off_lo), "r"(off_hi),
                             "r"(__float_as_int(w_lo)), "r"(__float_as_int(w_hi)) : "memory");
            const unsigned bm = __ballot_sync(0xffffffffu, any);
            const int r = (int)(key & 0xffffu), i = (int)((key >> 16) & 0x7fffu);
            const unsigned g_off = (unsigned)((r * PH + i / SR) * PW) * (unsigned)C + lane_ch;
#pragma unroll
            for (int pw = 0; pw < PW; ++pw)
                if ((bm >> (pw * SR)) & ((1u << SR) - 1u)) Acc<CPL>::ldg(dyt + (g_off + (unsigned)pw * (unsigned)C), G[pw]);
            return bm;
        };
        // B: apply the taps of one unit (records in stage buffer `slot`, gradients in G)
        auto stage_b = [&](int slot, const u64x (&G)[PW][HV], unsigned bm) {
#pragma unroll
            for (int j = 0; j < NX; ++j) {
                if (!((bm >> j) & 1u)) continue;
                int off_lo, off_hi, wl, wh;
                asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(off_lo), "=r"(off_hi), "=r"(wl), "=r"(wh)
                             : "r"(stage_s + slot * SB + j * 16));
                const unsigned a_lo = lane_acc + off_lo, a_hi = lane_acc + off_hi;
                const u64x w_lo = pack2(__int_as_float(wl), __int_as_float(wl)), w_hi = pack2(__int_as_float(wh), __int_as_float(wh));
                u64x v[HV], t[HV];
                // the two cells are distinct (or both the scratch cell): both read-modify-writes in flight together
                Acc<CPL>::ld(a_lo, v);
                Acc<CPL>::ld(a_hi, t);
#pragma unroll
                for (int q = 0; q < HV; ++q) { v[q] = fma2(G[j / SR][q], w_lo, v[q]); t[q] = fma2(G[j / SR][q], w_hi, t[q]); }
                Acc<CPL>::st(a_lo, v);
                Acc<CPL>::st(a_hi, t);
            }
        };

        // One batch of <= 32 units (lane = unit; `m` marks the lanes whose RoI overlaps this x-tile).  Software pipeline,
        // two register sets for the gradients:
        //   x-table entry of unit k+1 in flight | A(k): records + gradient loads | B(k-1): taps
        auto process_batch = [&](unsigned ux, unsigned uy, unsigned m) {
            u64x Ga[PW][HV], Gb[PW][HV];
            unsigned bma = 0u, bmb = 0u;
            unsigned key_n = 0u; float wy_n = 0.f; AxisEntry e_n = make_axis_zero();
            auto fetch_next = [&]() -> bool {
                if (m == 0u) return false;
                const int l = __ffs(m) - 1; m &= m - 1u;
                key_n = __shfl_sync(0xffffffffu, ux, l);
                wy_n = __uint_as_float(__shfl_sync(0xffffffffu, uy, l));
                if (lane < NX) e_n = xtab[(size_t)(key_n & 0xffffu) * NX + lane];
                return true;
            };
            fetch_next();
            unsigned key = key_n; float wy = wy_n; AxisEntry e = e_n;
            bool more = fetch_next();
            bma = stage_a(key, wy, e, 0, Ga);
            __syncwarp();
            for (;;) {
                if (!more) { stage_b(0, Ga, bma); break; }
                key = key_n; wy = wy_n; e = e_n; more = fetch_next();
                bmb = stage_a(key, wy, e, 1, Gb);
                stage_b(0, Ga, bma);
                __syncwarp();
                if (!more) { stage_b(1, Gb, bmb); break; }
                key = key_n; wy = wy_n; e = e_n; more = fetch_next();
                bma = stage_a(key, wy, e, 0, Ga);
                stage_b(1, Gb, bmb);
                __syncwarp();
            }
            __syncwarp();
        };

        // the row's own list, then (only when some row ran over its capacity) the shared overflow list
        const int row_cnt = min(zeroed[4 + row], row_cap), ovf_cnt = zeroed[1];
        const int row_pad = (row_cnt + 31) & ~31;                   // batches do not straddle the two lists
        const uint2* mine = row_list + (size_t)row * row_cap;
        for (int base = 0; base < row_pad + ovf_cnt; base += 32) {
            const int k = base + lane;
            uint2 u = make_uint2(0u, 0u);
            bool ov = false;
            if (k < row_cnt) { u = mine[k]; ov = true; }
            else if (k >= row_pad && k - row_pad < ovf_cnt) {
                const uint4 o = ovf[k - row_pad];
                u = make_uint2(o.x, o.y); ov = (int)o.z == row;
            }
            if (ov) {
                const int4 h = *reinterpret_cast<const int4*>(&roi_in[u.x & 0xffffu]);        // batch, x_lo, x_hi, y_lo
                ov = h.y <= x0 + kRowCells - 1 && h.z >= x0;
            }
            const unsigned m = __ballot_sync(0xffffffffu, ov);
            if (m) process_batch(u.x, u.y, m);
        }

        {   // write-out: lane = cell; CPL channels per shared load, one coalesced 128-byte row segment per channel
            const int x = x0 + lane;
            const bool ok = x < W;
            const unsigned rd = acc_s + lane * kCellBytes;
            char* p = reinterpret_cast<char*>(dx + (((size_t)n * C + (size_t)cb * CHB) * H + y) * W + x);
            const size_t cs = (size_t)H * W * sizeof(float);
#pragma unroll 4
            for (int c4 = 0; c4 < 32; ++c4) {
                u64x v[HV];
                Acc<CPL>::ld(rd + c4 * (CPL * 4), v);
#pragma unroll
                for (int q = 0; q < HV; ++q) {
                    float a, b; unpack2(v[q], a, b);
                    if (ok) { *reinterpret_cast<float*>(p) = a; *reinterpret_cast<float*>(p + cs) = b; }
                    p += 2 * cs;
                }
            }
        }
        __syncwarp();
    }
}

size_t roi_align_bwd_rows_workspace_bytes(int N, int R, int C, int H, int W, int PH, int PW, int sr) {
    RowsPlan p;
    return rows_plan(N, R, C, H, W, PH, PW, sr, &p) ? p.ws_bytes : 0;
}

template <int PW, int SR, int CPL, int WARPS>
static int launch_rows(const RowsPlan& p, unsigned char* ws, float* dx, int N, int C, int H, int W, int PH, cudaStream_t stream) {
    constexpr int NX = PW * SR;
    const size_t smem = (size_t)WARPS * rows_warp_smem<CPL, NX>();
    auto kern = roi_align_bwd_rows<PW, SR, CPL, WARPS>;
    if (const int rc = smem_opt_in(kern, smem)) return rc;
    int per_sm = 0;
    cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, WARPS * 32, smem);
    if (err != cudaSuccess) return (int)err;
    if (per_sm < 1) return kPathDeclined;
    const int items = N * H * p.tiles_x * (C / (32 * CPL));
    const int warps_needed = items;
    int grid = kNumSMs * per_sm;
    if (grid * WARPS > warps_needed) grid = (warps_needed + WARPS - 1) / WARPS;
    kern<<<grid, WARPS * 32, smem, stream>>>(
        reinterpret_cast<const BwdRoi*>(ws + p.roi_off), reinterpret_cast<const AxisEntry*>(ws + p.xtab_off),
        reinterpret_cast<int*>(ws + p.zero_off), reinterpret_cast<const uint2*>(ws + p.row_list_off), p.row_cap,
        reinterpret_cast<const uint4*>(ws + p.ovf_off), reinterpret_cast<const float*>(ws + p.dyt_off), dx, N, C, H, W, PH, p.tiles_x);
    return B200_ROI_OK;
}

// returns kPathDeclined when the path does not apply (caller falls back to another backward path)
int roi_align_backward_rows(const float* top_diff, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                            const float* rois, float* bottom_diff, const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    RowsPlan p;
    if (!rows_plan(N, R, C, H, W, PH, PW, sr, &p)) return kPathDeclined;
    if (workspace == nullptr || workspace_bytes < p.ws_bytes) return kPathDeclined;
    unsigned char* ws = (unsigned char*)workspace;
    const int bins = PH * PW;
    int tr_ch = kTransposeChannelsMax;                       // as many channels per CTA as fit ~100 KB (two CTAs per SM)
    while (tr_ch > 32 && (size_t)tr_ch * (bins | 1) * sizeof(float) > 100 * 1024) tr_ch >>= 1;
    if (tr_ch > C) tr_ch = (C + 31) / 32 * 32;
    const size_t smem_tr = (size_t)tr_ch * (bins | 1) * sizeof(float);
    if (smem_tr > 200 * 1024) return kPathDeclined;
    if (const int rc = smem_opt_in(roi_align_bwd_rows_tables, smem_tr)) return rc;
    cudaError_t err = cudaMemsetAsync(ws + p.zero_off, 0, p.zero_bytes, stream);    // item counter, overflow count, units per row
    if (err != cudaSuccess) return (int)err;
    const int cblocks = (C + tr_ch - 1) / tr_ch;
    const int table_ctas = (R * (p.ny + p.nx) + kTableThreads - 1) / kTableThreads;
    roi_align_bwd_rows_tables<<<table_ctas + R * cblocks, kTableThreads, smem_tr, stream>>>(
        rois, top_diff, scale, N, R, C, H, W, PH, PW, sr, table_ctas, tr_ch, reinterpret_cast<BwdRoi*>(ws + p.roi_off),
        reinterpret_cast<AxisEntry*>(ws + p.xtab_off), reinterpret_cast<int*>(ws + p.zero_off),
        reinterpret_cast<uint2*>(ws + p.row_list_off), p.row_cap, reinterpret_cast<uint4*>(ws + p.ovf_off),
        reinterpret_cast<float*>(ws + p.dyt_off), row_map);
    // channels per lane of the main kernel: 4 where PW == 7 and C % 128 == 0, else 2
    int rc;
    if (PW == 7) {
        if ((C % 128) == 0) rc = (sr == 1) ? launch_rows<7, 1, 4, 12>(p, ws, bottom_diff, N, C, H, W, PH, stream)
                                           : launch_rows<7, 2, 4, 12>(p, ws, bottom_diff, N, C, H, W, PH, stream);
        else rc = (sr == 1) ? launch_rows<7, 1, 2, 12>(p, ws, bottom_diff, N, C, H, W, PH, stream)
                            : launch_rows<7, 2, 2, 12>(p, ws, bottom_diff, N, C, H, W, PH, stream);
    } else {
        rc = (sr == 1) ? launch_rows<14, 1, 2, 12>(p, ws, bottom_diff, N, C, H, W, PH, stream)
                       : launch_rows<14, 2, 2, 12>(p, ws, bottom_diff, N, C, H, W, PH, stream);
    }
    if (rc != B200_ROI_OK) return rc;
    return finish_launch(2);
}

}  // namespace b200
