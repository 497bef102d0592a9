// roi_align_strip.cu -- Caffe2-exact RoIAlign FORWARD, "quad strip" fast path (round 2, second generation).
//
// Same decomposition as roi_align_stream.cu -- the map is cut into vertical strips, one persistent CTA per SM streams the
// rows of its piece of the (strip column, 32-channel group, row) space through a ring of row slots in shared memory, work
// = fragments (<= 8 bins of one bin row of one RoI, keyed by the first feature row they read) -- but everything that cost
// instructions there is organised differently:
//
//  * ring slot layout [column][32 channels] (cell = 128 B; 144 B = 128 + 16 pad in cp.async mode).  Compute mapping:
//    lane = (bin b = lane / 8, channel quad q = lane % 8): ONE LDS.128 fetches one bilinear tap for FOUR channels, a quarter
//    warp reads 128 contiguous bytes (conflict-free for any cell), the arithmetic works on channel pairs in 64-bit register
//    pairs, one scalar _rn instruction per half, so the reference's operation order is kept bit for bit.  A pass evaluates
//    4 bins x 32 channels.
//  * staging by TMA (default; W % 4 == 0 and a 16-byte aligned base): the map is described as the 4-D "x-quad" view
//    (x mod 4, n C + c, x div 4, y) -- strides (4 B, H W 4, 16 B, W 4), every load starting at innermost coordinate 0; a
//    plain (x, y, c) box would start unaligned at strip starts that are not 16-byte aligned and cannot put the channel
//    innermost -- and ONE cp.async.bulk.tensor.4d per row lands
//    [quad][channel][4 floats] in the slot's own memory, issued by lane 0 of the issuer warp as soon as the slot is free;
//    transposer warps (rows i mod T) wait for the slot's mbarrier, pull the row through registers (LDS.128, lane = channel)
//    and rewrite it IN PLACE as [column][channel] (STS.32, lane = channel), then publish next[t] = their first stream row
//    that has not landed.  128 shared-memory wavefronts per row instead of >= 512 LSU cycles for 64 four-byte cp.async;
//  * staging by cp.async (fallback: any W, e.g. FPN P5 with W = 42): every producer-side warp
//    stages rows i mod kPW with 4-byte LDGSTS, lane = column (full 128-byte lines per request: the L1 tracks outstanding
//    misses per line), the transposing write hits 8 distinct banks per returning sector (bank = 4 x + c with the 36-word
//    pitch); a warp's rows land in order (cp.async groups of one thread) and it publishes the same next[] word;
//  * residency is therefore min(next[]) -- one LDS.128 by a consumer warp whose fragment's last row is beyond what it has
//    already seen -- instead of a parity-tracked mbarrier wait per row and warp;
//  * slot release: every consumer warp publishes the stream index of the first row its current fragment reads (fragments
//    are sorted by key, a warp's marks never decrease); row i - K may be overwritten once the minimum over the published
//    words has passed it.  No per-row acquire / release, no phase bits;
//  * results leave registers directly (lane = 4 channels of one bin: four stores per pass, 16-byte runs of 4 bins), axis
//    tables are fetched per lane one fragment ahead straight into registers: no per-warp staging / table buffers, the
//    whole shared memory is ring;
//  * rows >= H are staged as zeros, and a sample clamped to the last row (low == high == H - 1, weights (1, 0)) reads
//    that zero row with weight 0: no slot is ever read before it was written, so the ring needs no zero-initialisation;
//  * prepass = ONE kernel (tables + fragment list, one returning atomic per fragment for its rank, grid barrier, CSR scan in
//    every CTA, fragment records at row pointer + rank, piece boundaries spread over the CTAs) instead of two kernels; the
//    main kernel is launched with programmatic dependent launch so that its prologue overlaps the tail of the prepass.
//
// Bit-exactness: every output element is computed by one lane in the reference's own operation order and written once;
// only bins whose samples cannot be resident together are cut into per-sample fragments accumulated with red.global.add
// onto zero-filled elements (<= 2 partial sums: order independent).
//
// Semantics: lib/modeling/roi_xfrom/roi_align/src/roi_align_kernel.cu (reference) :16-63, :65-121.
#include "common.cuh"
#include "strip_prep.cuh"
#include <cuda.h>                                              // CUtensorMap types only: the encoder is fetched with cudaGetDriverEntryPoint
#include <string.h>

namespace b200 {

namespace {

constexpr int kCW = 12;                                       // consumer warps (<= 32: their marks are read by one warp)
constexpr int kPW = 4;                                        // producer warps (stream row i is staged by warp i % kPW)
static_assert(kPW >= 2, "TMA staging needs an issuer warp and at least one transposer warp");
constexpr int kThreads = 32 * (kCW + kPW);
constexpr int kFragBins = 8;                                  // bins per fragment (two passes of 4)
// bytes per staged cell (template parameter CELL of the main kernel): 128 when rows are staged by TMA (the transposer writes
// 128 aligned bytes per column), 144 = 32 channels + 16 B pad with cp.async producers (bank = 4 x + c for the transposing write)
constexpr int kCellTma = 128, kCellAsync = 144;
constexpr int kDepth = 2;                                     // rows every producer warp keeps in flight
constexpr int kInflight = 8;                                  // TMA mode: rows issued but not yet transposed
constexpr int kMaxLevels = 6;
constexpr int kMaxCols = 96;
constexpr int kAxisMaxS = 32;
constexpr int kPrepThreads = 128;
constexpr int kMaxKeys = 6144;                                // CSR scan lives in shared memory
constexpr int kMaxK = 48;
constexpr unsigned kSmemBudget = 227u * 1024u;
constexpr unsigned kPrepSmemMax = 2 * (kMaxKeys + 1) * 4 + kAxisMaxS * kAxisMaxS * 12;     // strip_prep at the largest scan and fragment list
constexpr unsigned kFragCost = 10u, kPassCost = 9u;           // cost model of the partition (units ~ 10 instructions)
constexpr unsigned kRowCost = 44u;                            // cost of streaming one row in the same units

typedef unsigned long long u64;

struct StripLevel {
    const float* bottom;                                      // (N, C, H, W)
    float scale;
    int H, W, S;                                              // S: strips per image
    int q_base;                                               // its first strip column; column = q_base + image * S + strip
    int roi_begin;                                            // its first RoI (RoIs are stored level-major)
    int pad;
};

struct StripGeom {
    int N, R, C, PH, PW, sr;
    int ny, nx;
    int SX, WX, K, cell;                                      // columns per slot (8 XO), strip core width, ring depth, bytes per cell
    int L, Q, keys, G, pieces, max_entries, cap_r;            // cap_r: fragments one RoI can have at most
    StripLevel lv[kMaxLevels];
    int colstart[kMaxCols + 1];
};

__host__ __device__ __forceinline__ int level_of_roi(const StripGeom& g, int r) {
    int l = 0;
    while (l + 1 < g.L && r >= g.lv[l + 1].roi_begin) ++l;
    return l;
}

struct StripWs {
    uint4* ytab;                // [R][ny] {hy, ly, y_low, 0}
    uint4* xtab;                // [R][nx] {hx, lx, x_low * cell, 0}
    int* hist;                  // [keys]  fragments per key          (zero block)
    int* cost;                  // [keys]                             (zero block)
    int* maxend;                // [keys]                             (zero block)
    int* ticket;                // [4]                                (zero block)
    int* rowptr;                // [keys + 1]
    int* piece_start;           // [pieces + 1]
    uint2* entries;
    uint4* tmp;                 // [R][cap_r] {key index, rank within the key, record}: phase 1 -> phase 3 of the prepass
    int* tmpcnt;                // [R] fragments of the RoI (-1: batch index out of range)
};

// fragment record: x = r | ph << 16 | pw0 << 21 | (npw - 1) << 26 | red << 29 ; y = key | (end - key) << 16 | smask << 24
__device__ __forceinline__ uint2 pack_entry(int r, int ph, int pw0, int npw, int red, int key, int end, unsigned smask) {
    uint2 e;
    e.x = (unsigned)r | ((unsigned)ph << 16) | ((unsigned)pw0 << 21) | ((unsigned)(npw - 1) << 26) | ((unsigned)red << 29);
    e.y = (unsigned)key | ((unsigned)(end - key) << 16) | (smask << 24);
    return e;
}

struct AdjTap {
    int   low;
    float l, h;
};

// x axis: a sample on the last column (low = high = W - 1, weights (1, 0)) is read as cells (W - 2, W - 1) with weights
// (0, 1): the same sum term for term (the zero products do not change any finite partial sum); keeps both taps in the map.
__device__ __forceinline__ AdjTap adj_axis(float v, int size) {
    const AxisTap t = xfrom_axis(v, size);
    AdjTap a;
    a.low = t.low; a.l = t.l; a.h = t.h;
    if (t.low >= size - 1) { a.low = size - 2; a.l = 1.f; a.h = 0.f; }
    if (!t.valid) { a.l = 0.f; a.h = 0.f; }
    return a;
}

// Enumerate the fragments of bin row `ph` of one RoI.  yl: the reference's low tap row per y sample (a sample needs rows
// yl and yl + 1; row H is the zero row); xl: adjusted low cell per x sample.
// emit(strip, key, end, pw0, npw, smask, red, zero_owner)
template <int SR, class Emit>
__device__ __forceinline__ void enum_row(const int* yl, const int* xl, int ph, const StripGeom& g, int S, Emit&& emit) {
    const int i0 = ph * SR, i1 = i0 + SR - 1;
    int ngroups = 1;
    int key[2], end[2];
    unsigned ym[2];
    key[0] = yl[i0]; end[0] = yl[i1] + 2; ym[0] = (1u << SR) - 1u;
    key[1] = 0; end[1] = 0; ym[1] = 0;
    if (SR == 2 && end[0] - key[0] > g.K) {          // rows cannot be resident together: one fragment per y sample
        ngroups = 2;
        end[0] = yl[i0] + 2; ym[0] = 1u;
        key[1] = yl[i1]; end[1] = yl[i1] + 2; ym[1] = 2u;
    }
    constexpr unsigned kXFull = (1u << SR) - 1u;
    for (int gi = 0; gi < ngroups; ++gi) {
        int run_s = -1, run_pw0 = 0, run_n = 0;
        unsigned run_xm = 0;
        auto flush = [&]() {
            if (run_n == 0) return;
            unsigned smask;
            if (SR == 1) smask = 1u;
            else smask = ((ym[gi] & 1u) ? run_xm : 0u) | ((ym[gi] & 2u) ? (run_xm << 2) : 0u);
            const bool red = (ym[gi] != kXFull) || (run_xm != kXFull);
            const bool owner = red && (ym[gi] & 1u) && (run_xm & 1u);
            emit(run_s, key[gi], end[gi], run_pw0, run_n, smask, red ? 1 : 0, owner);
            run_n = 0;
        };
        auto push = [&](int s, unsigned xm, int pw) {
            if (run_n > 0 && s == run_s && xm == run_xm && run_n < kFragBins && pw == run_pw0 + run_n) { ++run_n; return; }
            flush();
            run_s = s; run_xm = xm; run_pw0 = pw; run_n = 1;
        };
        for (int pw = 0; pw < g.PW; ++pw) {
            const int j0 = pw * SR, j1 = j0 + SR - 1;
            const int s0 = min(xl[j0] / g.WX, S - 1);
            if (SR == 1 || xl[j1] + 1 <= s0 * g.WX + g.SX - 1) {
                push(s0, kXFull, pw);
            } else {                                   // x samples in different strips: one fragment per x sample
                push(s0, 1u, pw);
                push(min(xl[j1] / g.WX, S - 1), 2u, pw);
            }
        }
        flush();
    }
}

// ------------------------------------------------------------------------------------------------
// prepass (one launch): tables + histogram | grid barrier | CSR scan (every CTA) | records, zero-fill, pieces
// ------------------------------------------------------------------------------------------------
template <int SR>
__global__ void __launch_bounds__(kPrepThreads)
strip_prep(const float* __restrict__ rois, StripGeom g, StripWs ws, float* __restrict__ out, const int* __restrict__ row_map) {
    extern __shared__ unsigned s_dyn[];                       // [keys + 1] fragment prefix, [keys + 1] cost prefix, [cap_r][3] fragment list
    __shared__ int s_nlist;
    __shared__ int s_yl[kAxisMaxS], s_xl[kAxisMaxS];
    __shared__ unsigned short s_zero[kAxisMaxS * kAxisMaxS];
    __shared__ int s_nzero;
    __shared__ unsigned s_ph[kPrepThreads], s_pc[kPrepThreads];
    const int t = threadIdx.x;
    const int keys = g.keys;
    unsigned* s_pre = s_dyn;
    unsigned* s_cpre = s_dyn + (keys + 1);
    unsigned* s_list = s_dyn + 2 * (keys + 1);               // {key index, record.x, record.y} per fragment of the current RoI

    auto axes = [&](int r, bool write_tables) -> XfromRoi {   // per-RoI axis tables (all IEEE divisions live here)
        const StripLevel& lv = g.lv[level_of_roi(g, r)];
        const XfromRoi geo = xfrom_roi(rois + 5 * (size_t)r, lv.scale, g.PH, g.PW, g.sr);
        if (t < g.ny + g.nx) {
            const bool isy = t < g.ny;
            const int s = isy ? t : t - g.ny;
            if (isy) {
                const AxisTap a = xfrom_axis(xfrom_coord(geo.start_h, geo.bin_h, s / SR, s % SR, SR), lv.H);
                s_yl[s] = a.low;
                if (write_tables) {
                    uint4 e;
                    e.x = __float_as_uint(a.valid ? a.h : 0.f); e.y = __float_as_uint(a.valid ? a.l : 0.f);
                    e.z = (unsigned)a.low; e.w = 0u;
                    ws.ytab[(size_t)r * g.ny + s] = e;
                }
            } else {
                const AdjTap a = adj_axis(xfrom_coord(geo.start_w, geo.bin_w, s / SR, s % SR, SR), lv.W);
                s_xl[s] = a.low;
                if (write_tables) {
                    uint4 e;
                    e.x = __float_as_uint(a.h); e.y = __float_as_uint(a.l);
                    e.z = (unsigned)(a.low * g.cell); e.w = 0u;
                    ws.xtab[(size_t)r * g.nx + s] = e;
                }
            }
        }
        return geo;
    };

    // ---- phase 1: tables; the RoI's fragments are listed in shared memory by the bin-row threads, then ALL threads take one
    // fragment each: rank within its key (the returning atomic's latency is paid once and hides behind the grid barrier),
    // cost / extent atomics, and a temporary record that phase 3 only has to drop into the CSR
    for (int r = blockIdx.x; r < g.R; r += gridDim.x) {
        __syncthreads();                                      // s_yl / s_xl / s_list of the previous RoI are no longer read
        const XfromRoi geo = axes(r, true);
        if (t == 0) s_nlist = 0;
        __syncthreads();
        const StripLevel& lv = g.lv[level_of_roi(g, r)];
        const bool batch_ok = geo.batch >= 0 && geo.batch < g.N;
        if (batch_ok && t < g.PH) {
            const int cbase = lv.q_base + geo.batch * lv.S;
            enum_row<SR>(s_yl, s_xl, t, g, lv.S, [&](int s, int key, int end, int pw0, int npw, unsigned smask, int red, bool owner) {
                const int idx = atomicAdd(&s_nlist, 1);
                const uint2 e = pack_entry(r, t, pw0, npw, red, key, end, smask);
                s_list[3 * idx] = (unsigned)(g.colstart[cbase + s] + key); s_list[3 * idx + 1] = e.x; s_list[3 * idx + 2] = e.y;
                (void)owner;
            });
        }
        __syncthreads();
        const int n = s_nlist;
        for (int idx = t; idx < n; idx += kPrepThreads) {
            const unsigned k = s_list[3 * idx], ex = s_list[3 * idx + 1], ey = s_list[3 * idx + 2];
            const int npw = (int)((ex >> 26) & 7u) + 1, end = (int)(ey & 0xffffu) + (int)((ey >> 16) & 0xffu);
            const int rank = atomicAdd(&ws.hist[k], 1);
            atomicAdd(&ws.cost[k], (int)(kFragCost + kPassCost * (unsigned)((npw + 3) >> 2)));
            atomicMax(&ws.maxend[k], end);
            ws.tmp[(size_t)r * g.cap_r + idx] = make_uint4(k, (unsigned)rank, ex, ey);
        }
        if (t == 0) ws.tmpcnt[r] = batch_ok ? n : -1;
    }
    // ---- grid barrier (the grid is sized to be resident: see the launcher)
    prepass::grid_barrier(ws.ticket);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");      // the main kernel may start its prologue
    // ---- phase 2: exclusive prefix of the fragment histogram and of the cost, in every CTA's shared memory
    prepass::scan_keys<kPrepThreads>(ws.hist, ws.cost, kRowCost, keys, s_pre, s_cpre, s_ph, s_pc);
    // row pointers for the main kernel: every CTA writes a slice
    for (int k = blockIdx.x * kPrepThreads + t; k <= keys; k += gridDim.x * kPrepThreads) ws.rowptr[k] = (int)s_pre[k];
    // piece boundaries: every CTA holds the whole prefix, so they are spread over the grid (one per CTA, thread 0)
    if (t == 0)
        for (int p = blockIdx.x; p <= g.pieces; p += gridDim.x)
            ws.piece_start[p] = prepass::piece_start(p, g.pieces, g.G, keys, g.Q, g.colstart, s_cpre);
    // ---- phase 3: fragment records into the CSR (position = row pointer + rank); zero-fill of the elements that are
    // accumulated with red.add (the bins of the fragments that hold a split bin's first sample)
    const int bins = g.PH * g.PW;
    for (int r = blockIdx.x; r < g.R; r += gridDim.x) {
        __syncthreads();
        if (t == 0) s_nzero = 0;
        __syncthreads();
        const int n = __ldcg(&ws.tmpcnt[r]);
        if (n >= 0) {
            for (int idx = t; idx < n; idx += kPrepThreads) {
                const uint4 rec = __ldcg(&ws.tmp[(size_t)r * g.cap_r + idx]);
                const int pos = (int)s_pre[rec.x] + (int)rec.y;
                if (pos < g.max_entries) ws.entries[pos] = make_uint2(rec.z, rec.w);
                const bool owner = ((rec.z >> 29) & 1u) && ((rec.w >> 24) & 1u);
                if (owner) {
                    const int ph = (rec.z >> 16) & 31u, pw0 = (rec.z >> 21) & 31u, npw = (int)((rec.z >> 26) & 7u) + 1;
                    const int z = atomicAdd(&s_nzero, npw);
                    for (int i = 0; i < npw; ++i) s_zero[z + i] = (unsigned short)(ph * g.PW + pw0 + i);
                }
            }
        } else {
            for (int i = t; i < bins; i += kPrepThreads) s_zero[i] = (unsigned short)i;       // the reference would read out of bounds
            if (t == 0) s_nzero = bins;
        }
        __syncthreads();
        const int nz = s_nzero;
        if (nz > 0) {
            float* out_r = out + (size_t)(row_map ? row_map[r] : r) * g.C * bins;
            for (int idx = t; idx < g.C * nz; idx += kPrepThreads) {
                const int c = idx / nz, k = idx - c * nz;
                out_r[(size_t)c * bins + s_zero[k]] = 0.f;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// main kernel helpers
// ------------------------------------------------------------------------------------------------
__device__ u64* g_strip_dead = nullptr;                       // optional host-pinned watchdog records ([CTA][32] u64)

__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async4(unsigned dst, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async4_if(unsigned dst, const float* src, bool ok) {      // !ok: zero-fill
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(ok ? 4 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ int lds_acquire(unsigned addr) {
    int v;
    asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ int4 lds_acquire4(unsigned addr) {
    int4 v;
    asm volatile("ld.acquire.cta.shared.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void sts_release(unsigned addr, int v) {
    asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// ---- mbarrier + TMA (row staging through the tensor-memory accelerator) ----
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned bar, unsigned parity) {
    unsigned ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"     // %3: the hardware may park the thread this long (ns)
        "selp.u32 %0, 1, 0, p;\n"
        "}" : "=r"(ok) : "r"(bar), "r"(parity), "r"(10000u) : "memory");
    return ok != 0;
}
// One row of one (image, strip, 32-channel group) as a 4-D box (4 columns, 32 channels, SX / 4 column quads, 1 row) of the
// x-quad view of the map: lands as [quad][channel][4 floats]; rows / quads / channels beyond the map are zero-filled.
__device__ __forceinline__ void tma_load_row(unsigned dst, const CUtensorMap* map, unsigned bar, int chan, int xquad, int y) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(dst), "l"((u64)map), "r"(bar), "r"(0), "r"(chan), "r"(xquad), "r"(y) : "memory");
}

// Low-water marks are published with a plain volatile store: shared-memory instructions of one warp are performed in program
// order, so the store cannot overtake the (converged, __syncwarp'ed) tap loads that precede it -- a release fence here would
// also wait for the fragment's global stores (MEMBAR per fragment).
__device__ __forceinline__ void sts_volatile(unsigned addr, int v) {
    asm volatile("st.volatile.shared.s32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void watchdog_note(unsigned tag, u64 info) {
    if (g_strip_dead != nullptr && (threadIdx.x & 31) == 0) {
        g_strip_dead[blockIdx.x * 32 + (threadIdx.x >> 5)] = 0xDEAD000000000000ull | ((u64)tag << 40) | (info & 0xffffffffffull);
        __threadfence_system();
    }
}

// fp32 pairs in one 64-bit register pair (the shape of the 128-bit shared loads).  sm_90 has no packed fp32x2
// instructions: each operation is two scalar IEEE-754 RN instructions, one per half.
__device__ __forceinline__ u64 pack2f(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void unpack2f(u64 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
    float a0, a1, b0, b1; unpack2f(a, a0, a1); unpack2f(b, b0, b1);
    return pack2f(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
    float a0, a1, b0, b1; unpack2f(a, a0, a1); unpack2f(b, b0, b1);
    return pack2f(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
    float a0, a1, b0, b1, c0, c1; unpack2f(a, a0, a1); unpack2f(b, b0, b1); unpack2f(c, c0, c1);
    return pack2f(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

struct Quad { u64 lo, hi; };                                  // four channels of one tap
template <int OFF>
__device__ __forceinline__ Quad lds_quad(unsigned at) {
    Quad v;
    asm volatile("ld.shared.v2.b64 {%0, %1}, [%2+%3];" : "=l"(v.lo), "=l"(v.hi) : "r"(at), "n"(OFF));
    return v;
}

// The four taps of one sample for this lane's four channels: rows (slot, next slot) x cells (x_low, x_low + 1).
template <int RB, int CELL>
struct Taps4 {
    Quad v1, v2, v3, v4;
    __device__ __forceinline__ void load(unsigned at) {
        v1 = lds_quad<0>(at); v2 = lds_quad<CELL>(at); v3 = lds_quad<RB>(at); v4 = lds_quad<RB + CELL>(at);
    }
};

// One bilinear sample, the reference's rounding recipe per channel:
// val = FFMA(v4, w4, FFMA(v3, w3, FFMA(v1, w1, FMUL(v2, w2)))), w1 = hy*hx, w2 = hy*lx, w3 = ly*hx, w4 = ly*lx;
// then acc = FADD(acc, val).  hh / ll: (hy, hy) / (ly, ly); xh / xl: (hx, hx) / (lx, lx).
template <int RB, int CELL>
__device__ __forceinline__ void sample_acc(const Taps4<RB, CELL>& t, u64 hh, u64 ll, u64 xh, u64 xl, u64& acc_lo, u64& acc_hi) {
    const u64 w1 = mul2(hh, xh), w2 = mul2(hh, xl), w3 = mul2(ll, xh), w4 = mul2(ll, xl);
    acc_lo = add2(acc_lo, fma2(t.v4.lo, w4, fma2(t.v3.lo, w3, fma2(t.v1.lo, w1, mul2(t.v2.lo, w2)))));
    acc_hi = add2(acc_hi, fma2(t.v4.hi, w4, fma2(t.v3.hi, w3, fma2(t.v1.hi, w1, mul2(t.v2.hi, w2)))));
}

struct StripArgs {
    const uint4* ytab;
    const uint4* xtab;
    const uint2* entries;
    const int* rowptr;
    const int* maxend;
    const int* piece_start;
    float* out;
    const int* row_map;
    int C, G, K, WX, PH, PW, ny, nx, L, Q;
    unsigned magicK;                                          // floor(2^32 / K) + 1: i / K == umulhi(i, magicK) for i < 2^32 / K
    int tma;                                                  // rows are staged by TMA + transposer warps (else: cp.async producers)
    StripLevel lv[kMaxLevels];
    int colstart[kMaxCols + 1];
};

struct alignas(64) StripMaps {
    CUtensorMap m[kMaxLevels];                                // x-quad view of every level's feature map (TMA mode)
};

struct Item {
    int lvl, n, s, g, ya, yb, e0, e1, yhi, kbase;
};

// Decode the item that starts at linear index L (all lanes of the calling warp; yhi by warp reduction).
__device__ __forceinline__ Item decode_item(int L, int L1, const StripArgs& a, int lane) {
    Item it;
    int lo = 0, hi = a.Q - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.G * a.colstart[mid] <= L) lo = mid; else hi = mid - 1;
    }
    const int q = lo;
    it.kbase = a.colstart[q];
    const int Hq = a.colstart[q + 1] - it.kbase;
    const int rem = L - a.G * it.kbase;
    it.g = rem / Hq;
    it.ya = rem - it.g * Hq;
    it.yb = min(Hq, it.ya + (L1 - L));
    int l = 0;
    while (l + 1 < a.L && q >= a.lv[l + 1].q_base) ++l;
    it.lvl = l;
    const int qq = q - a.lv[l].q_base;
    it.n = qq / a.lv[l].S;
    it.s = qq - it.n * a.lv[l].S;
    it.e0 = __ldg(&a.rowptr[it.kbase + it.ya]);
    it.e1 = __ldg(&a.rowptr[it.kbase + it.yb]);
    int m = 0;
    if (it.e1 > it.e0) {
        for (int y = it.ya + lane; y < it.yb; y += 32) m = max(m, __ldg(&a.maxend[it.kbase + y]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    it.yhi = m;
    return it;
}

// Stage row y of one (image, strip, channel group) into a ring slot.  lane = column within a 32-column chunk: every request
// reads 128 contiguous bytes of one channel row (one or two cache lines -- the L1 tracks outstanding misses per line, so a
// request that gathered four channels x 32 bytes keeps four times fewer bytes in flight); the transposing
// write of each returning 32-byte sector hits 8 distinct banks (bank = 4 x + c with the 36-word cell pitch).
// src: (channel c0, row y, column x0 + lane); dst: slot + lane * CELL.
template <int XO, int CELL>
__device__ __forceinline__ void stage_row(const float* __restrict__ src, size_t plane, unsigned dst, bool interior, bool row_ok,
                                          int xw, int cvalid, int lane) {
    constexpr int M = XO / 4;                                  // 32-column chunks
    if (interior) {
#pragma unroll 8
        for (int c = 0; c < 32; ++c) {
#pragma unroll
            for (int m = 0; m < M; ++m) cp_async4(dst + (unsigned)(m * 32 * CELL + c * 4), src + 32 * m);
            src += plane;
        }
    } else {
#pragma unroll 4
        for (int c = 0; c < 32; ++c) {
            const bool cok = row_ok && c < cvalid;
            const float* p = src + (size_t)(cok ? c : 0) * plane;
#pragma unroll
            for (int m = 0; m < M; ++m) {
                const bool ok = cok && (32 * m + lane) < xw;
                cp_async4_if(dst + (unsigned)(m * 32 * CELL + c * 4), ok ? p + 32 * m : src, ok);
            }
        }
    }
}

template <int SR>
struct FragTab {
    uint4 x[2][SR];                                           // [pass][x sample] of this lane's bin
    uint4 y[SR];
};

template <int SR, int XO, int CELL>
__global__ void __launch_bounds__(kThreads, 1)
roi_align_strip_fwd(const __grid_constant__ StripMaps maps, const StripArgs a) {
    constexpr int SX = 8 * XO;
    constexpr int RB = SX * CELL;                                 // bytes of one ring slot
    extern __shared__ unsigned char smem_raw[];
    const unsigned ring = (smem_addr(smem_raw) + 127u) & ~127u;
    // ring: K logical slots + a mirror of slot 0 behind slot K - 1 (row y + 1 is always the next physical slot)
    // control words: pub[32] (consumer low-water marks); next[kPW] (per producer: stream index of its first row not yet landed)
    const unsigned ctl = ring + (unsigned)(a.K + 1) * (unsigned)RB;
    const unsigned pub = ctl, next_addr = ctl + 128u, full_bar = ctl + 256u;       // full_bar[K]: TMA completion per slot
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (a.tma && tid == 0) {
        for (int k = 0; k < a.K; ++k) mbar_init(full_bar + 8u * k, 1u);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    if (tid < kCW) sts_release(pub + 4u * tid, 0);
    if (tid >= kCW && tid < kCW + 4) {                         // next[w]: cp.async mode: producer w; TMA mode: transposer w (warp kCW + 1 + w)
        const int w = tid - kCW;
        sts_release(next_addr + 4u * w, w < (a.tma ? kPW - 1 : kPW) ? w : 0x7fffffff);
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");             // the prepass's results are visible from here on
    // NOT __ldg: a read-only (.nc) load carries no dependence on the wait above and was hoisted to the top of the kernel,
    // where the prepass had not written the piece table yet (stale / garbage piece bounds on a fresh workspace)
    int L0, L1;
    asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(L0) : "l"(a.piece_start + blockIdx.x) : "memory");
    asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(L1) : "l"(a.piece_start + blockIdx.x + 1) : "memory");

    if (warp >= kCW && a.tma) {
        // =============================== TMA issuer + transposers ===============================
        // Warp kCW issues ONE cp.async.bulk.tensor per row (lane 0) as soon as the slot is free -- the whole free part of the
        // ring is in flight, at no LSU cost.  The box lands as [column quad][channel][4 columns] in the slot's own memory;
        // transposer warp t (rows i % T == t) waits for the slot's mbarrier, pulls the row through its registers (LDS.128,
        // lane = channel: 512 contiguous bytes per request) and rewrites it IN PLACE as [column][channel] with the 36-word
        // cell pitch CELL (STS.32, lane = channel: 128 contiguous bytes), in batches of 32 columns, highest first -- a cell's new
        // place (CELL x >= 128 x) is never below the not yet read part of the row -- then publishes next[t] like a cp.async producer.
        constexpr int T = kPW - 1;
        constexpr unsigned kRowBytes = (unsigned)SX * 128u;
        const int role = warp - kCW;                           // 0: issuer, 1 .. T: transposers
        int i = 0, slot = 0, turn = 0;
        int low_c = 0, low_t = 0;                              // issuer: last observed minimum of the consumer / transposer marks
        unsigned use_parity = 0;                               // parity of the current use of `slot` = (i / K) & 1
        for (int L = L0; L < L1;) {
            const Item it = decode_item(L, L1, a, lane);
            L += it.yb - it.ya;
            if (it.e1 <= it.e0) continue;
            const int chan = it.n * a.C + it.g * 32;
            const int xquad = (it.s * a.WX) >> 2;
            for (int y = it.ya; y < it.yhi; ++y) {
                if (role == 0) {
                    // row i - K must be done with by every consumer (and transposed); at most kInflight rows are kept between issue
                    // and transposition: the first rows a piece needs do not queue behind a ring-full of later ones in DRAM
                    if ((i >= a.K && low_c <= i - a.K) || (i >= kInflight && low_t <= i - kInflight)) {
                        unsigned spins = 0;
                        for (;;) {
                            const int vc = lane < kCW ? lds_acquire(pub + 4u * lane) : 0x7fffffff;
                            const int vt = lane < T ? lds_acquire(next_addr + 4u * lane) : 0x7fffffff;
                            low_t = __reduce_min_sync(0xffffffffu, vt);
                            low_c = min(__reduce_min_sync(0xffffffffu, vc), low_t);
                            if (low_c > i - a.K && low_t > i - kInflight) break;
                            __nanosleep(60);
                            if (++spins == (1u << 21)) watchdog_note(3u, ((u64)(unsigned)i << 20) | (u64)(unsigned)low_c);
                            if (spins > (1u << 22)) __trap();
                        }
                    }
                    if (lane == 0) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy accesses of the slot are done
                        const unsigned bar = full_bar + 8u * slot;
                        mbar_expect_tx(bar, kRowBytes);
                        tma_load_row(ring + (unsigned)slot * (unsigned)RB, &maps.m[it.lvl], bar, chan, xquad, y);
                    }
                } else if (turn == role - 1) {
                    const unsigned bar = full_bar + 8u * slot;
                    if (!mbar_try_wait(bar, use_parity)) {
                        unsigned spins = 0;
                        while (!mbar_try_wait(bar, use_parity)) {
                            if (++spins == (1u << 19)) watchdog_note(4u, ((u64)(unsigned)i << 20) | (u64)slot);
                            if (spins > (1u << 20)) __trap();
                        }
                    }
                    const unsigned sbase = ring + (unsigned)slot * (unsigned)RB;
                    const unsigned rd = sbase + (unsigned)lane * 16u, wr = sbase + (unsigned)lane * 4u;
                    const unsigned wr2 = ring + (unsigned)a.K * (unsigned)RB + (unsigned)lane * 4u;      // mirror of slot 0
#pragma unroll
                    for (int q0 = SX / 4 - 8; q0 >= 0; q0 -= 8) {                // 8 column quads (32 columns) per batch, highest first
                        uint4 v[8];
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v[j].x), "=r"(v[j].y), "=r"(v[j].z), "=r"(v[j].w) : "r"(rd + (unsigned)((q0 + j) * 512)));
                        __syncwarp();                                              // every lane has read the batch before any lane overwrites it
#pragma unroll
                        for (int j = 7; j >= 0; --j) {
                            const unsigned o = (unsigned)((q0 + j) * 4 * CELL);
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(wr + o), "r"(v[j].x) : "memory");
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(wr + o + CELL), "r"(v[j].y) : "memory");
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(wr + o + 2 * CELL), "r"(v[j].z) : "memory");
                            asm volatile("st.shared.b32 [%0], %1;" ::"r"(wr + o + 3 * CELL), "r"(v[j].w) : "memory");
                            if (slot == 0) {
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(wr2 + o), "r"(v[j].x) : "memory");
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(wr2 + o + CELL), "r"(v[j].y) : "memory");
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(wr2 + o + 2 * CELL), "r"(v[j].z) : "memory");
                                asm volatile("st.shared.b32 [%0], %1;" ::"r"(wr2 + o + 3 * CELL), "r"(v[j].w) : "memory");
                            }
                        }
                        __syncwarp();
                    }
                    __threadfence_block();
                    __syncwarp();
                    if (lane == 0) sts_release(next_addr + 4u * (role - 1), i + T);
                }
                ++i;
                if (++slot == a.K) { slot = 0; use_parity ^= 1u; }
                if (++turn == T) turn = 0;
            }
        }
        if (role > 0) {
            __syncwarp();
            if (lane == 0) sts_release(next_addr + 4u * (role - 1), 0x7fffffff);
        }
        return;
    }
    if (warp >= kCW) {
        // =============================== producers (cp.async mode) ===============================
        // Stream row i (all items of the piece, in order) is staged by producer warp i % kPW.  A warp's rows land in order
        // (cp.async groups of one thread), so it publishes next = the stream index of its first row that has not landed;
        // rows [0, min over the producers of next) are resident.
        const int pw = warp - kCW;
        const unsigned my_next = next_addr + 4u * pw;
        int i = 0, slot = 0, turn = 0;                         // stream row index, its slot (i % K), i % kPW
        int committed = 0, landed = 0;                         // this warp's rows: staged / known to have landed
        int minpub = 0;                                        // last observed minimum of the consumers' marks
        for (int L = L0; L < L1;) {
            const Item it = decode_item(L, L1, a, lane);
            L += it.yb - it.ya;
            if (it.e1 <= it.e0) continue;
            const StripLevel& lv = a.lv[it.lvl];
            const size_t plane = (size_t)lv.H * lv.W;
            const int x0 = it.s * a.WX;
            const int c0 = it.g * 32;
            const int cvalid = min(32, a.C - c0);
            const int xw = lv.W - x0;
            const bool full = cvalid == 32 && xw >= SX;
            const float* src = lv.bottom + ((size_t)it.n * a.C + c0) * plane + (size_t)it.ya * lv.W + x0 + (lane < xw ? lane : 0);
            for (int y = it.ya; y < it.yhi; ++y) {
                if (turn == pw) {
                    if (i >= a.K && minpub <= i - a.K) {
                        // the slot still holds row i - K: everything this warp committed must be visible before it blocks
                        cp_async_wait<0>();
                        __threadfence_block();
                        __syncwarp();
                        if (landed < committed) { landed = committed; if (lane == 0) sts_release(my_next, pw + landed * kPW); }
                        unsigned spins = 0;
                        for (;;) {
                            const int v = lane < kCW ? lds_acquire(pub + 4u * lane) : 0x7fffffff;
                            minpub = __reduce_min_sync(0xffffffffu, v);
                            if (minpub > i - a.K) break;
                            __nanosleep(100);
                            if (++spins == (1u << 21)) watchdog_note(1u, ((u64)(unsigned)i << 20) | (u64)(unsigned)minpub);
                            if (spins > (1u << 22)) __trap();
                        }
                    }
                    const bool row_ok = y < lv.H;
                    const float* srow = src + (size_t)(row_ok ? y - it.ya : 0) * lv.W;
                    const unsigned dst = ring + (unsigned)slot * (unsigned)RB + (unsigned)(lane * CELL);
                    stage_row<XO, CELL>(srow, plane, dst, full && row_ok, row_ok, xw, cvalid, lane);
                    if (slot == 0)
                        stage_row<XO, CELL>(srow, plane, ring + (unsigned)a.K * (unsigned)RB + (unsigned)(lane * CELL), full && row_ok, row_ok, xw, cvalid, lane);
                    cp_async_commit();
                    ++committed;
                    if (committed - landed > kDepth) {             // all but this warp's kDepth newest rows have landed
                        cp_async_wait<kDepth>();
                        __threadfence_block();
                        __syncwarp();
                        landed = committed - kDepth;
                        if (lane == 0) sts_release(my_next, pw + landed * kPW);
                    }
                }
                ++i;
                if (++slot == a.K) slot = 0;
                if (++turn == kPW) turn = 0;
            }
        }
        cp_async_wait<0>();
        __threadfence_block();
        __syncwarp();
        if (lane == 0) sts_release(my_next, 0x7fffffff);
        return;
    }

    // =============================== consumers ===============================
    const int b = lane >> 3, q = lane & 7;
    const int bins = a.PH * a.PW;
    constexpr float kInvCount = 1.f / (float)(SR * SR);
    const u64 inv2 = pack2f(kInvCount, kInvCount);
    const u64 zero2 = pack2f(0.f, 0.f);
    int ready_c = 0;                                           // cached: rows [0, ready_c) of the stream are resident
    int ibase = 0;                                             // stream index of the current item's first row

    auto load_tab = [&](const uint2& en) -> FragTab<SR> {
        FragTab<SR> tb;
        const int rn = en.x & 0xffffu, phn = (en.x >> 16) & 31u, pwn = (en.x >> 21) & 31u, nn = (int)((en.x >> 26) & 7u) + 1;
        const uint4* xr = a.xtab + (size_t)rn * a.nx;
        const int bA = pwn + min(b, nn - 1), bB = pwn + min(4 + b, nn - 1);
#pragma unroll
        for (int s = 0; s < SR; ++s) {
            tb.x[0][s] = __ldg(xr + bA * SR + s);
            tb.x[1][s] = __ldg(xr + bB * SR + s);
            tb.y[s] = __ldg(a.ytab + (size_t)rn * a.ny + phn * SR + s);
        }
        return tb;
    };

    for (int L = L0; L < L1;) {
        const Item it = decode_item(L, L1, a, lane);
        L += it.yb - it.ya;
        if (it.e1 <= it.e0) continue;
        const unsigned lane_base = ring + (unsigned)(q * 16) - (unsigned)(it.s * a.WX * CELL);
        const int c0 = it.g * 32;
        const int cq = c0 + 4 * q;                             // this lane's first channel
        const int irel = ibase - it.ya;                        // stream index of row y = irel + y

        int e = it.e0 + warp;
        uint2 ent0 = make_uint2(0u, 0u), ent1 = make_uint2(0u, 0u);
        FragTab<SR> tnext;
        if (e < it.e1) { ent0 = __ldg(&a.entries[e]); tnext = load_tab(ent0); }
        if (e + kCW < it.e1) ent1 = __ldg(&a.entries[e + kCW]);
        while (e < it.e1) {
            const uint2 cur = ent0;
            const FragTab<SR> tb = tnext;
            const int e_next = e + kCW;
            ent0 = ent1;
            if (e_next < it.e1) tnext = load_tab(ent0);                             // in flight while this fragment computes
            if (e_next + kCW < it.e1) ent1 = __ldg(&a.entries[e_next + kCW]);
            const int r = cur.x & 0xffffu, ph = (cur.x >> 16) & 31u, pw0 = (cur.x >> 21) & 31u;
            const int npw = (int)((cur.x >> 26) & 7u) + 1;
            const bool red = (cur.x >> 29) & 1u;
            const int key = cur.y & 0xffffu, end = key + (int)((cur.y >> 16) & 0xffu);
            const unsigned smask = (cur.y >> 24) & 0xfu;
            // publish the low-water mark (all lanes are past the previous fragment's last shared-memory read), then make sure
            // rows [key, end) are resident
            __syncwarp();
            if (lane == 0) sts_volatile(pub + 4u * warp, irel + key);
            const int i_last = irel + end - 1;
            if (i_last >= ready_c) {
                unsigned spins = 0;
                for (;;) {
                    const int4 nx4 = lds_acquire4(next_addr);
                    ready_c = min(min(nx4.x, nx4.y), min(nx4.z, nx4.w));
                    if (ready_c > i_last) break;
                    __nanosleep(a.tma ? 64u : 200u);           // cp.async mode: a starved consumer must not crowd the producers' LDGSTS out of the MIO queue
                    if (++spins == (1u << 20)) watchdog_note(2u, ((u64)(unsigned)i_last << 20) | (u64)(unsigned)ready_c);
                    if (spins > (1u << 21)) __trap();
                }
            }
            // row bases (uniform): slot of y_low; the lower tap row is the next physical slot
            unsigned rt[SR];
            u64 hh[SR], ll[SR];
#pragma unroll
            for (int s = 0; s < SR; ++s) {
                const unsigned iy = (unsigned)(irel + (int)tb.y[s].z);
                const unsigned sl = iy - __umulhi(iy, a.magicK) * (unsigned)a.K;
                rt[s] = lane_base + sl * (unsigned)RB;
                hh[s] = pack2f(__uint_as_float(tb.y[s].x), __uint_as_float(tb.y[s].x));
                ll[s] = pack2f(__uint_as_float(tb.y[s].y), __uint_as_float(tb.y[s].y));
            }
            const int orow = a.row_map ? __ldg(&a.row_map[r]) : r;
            float* obase = a.out + ((size_t)orow * a.C + cq) * bins + ph * a.PW + pw0 + b;
#pragma unroll
            for (int pass = 0; pass < 2; ++pass) {
                if (4 * pass + b < npw) {
                    u64 acc_lo = zero2, acc_hi = zero2;
                    u64 xh[SR], xl[SR];
                    unsigned xo[SR];
#pragma unroll
                    for (int s = 0; s < SR; ++s) {
                        xh[s] = pack2f(__uint_as_float(tb.x[pass][s].x), __uint_as_float(tb.x[pass][s].x));
                        xl[s] = pack2f(__uint_as_float(tb.x[pass][s].y), __uint_as_float(tb.x[pass][s].y));
                        xo[s] = tb.x[pass][s].z;
                    }
                    if (SR == 1) {
                        Taps4<RB, CELL> t0; t0.load(rt[0] + xo[0]);
                        sample_acc<RB, CELL>(t0, hh[0], ll[0], xh[0], xl[0], acc_lo, acc_hi);
                    } else if (smask == 0xfu) {
                        // whole bins (the common case): all 16 taps are requested before the first one is used
                        Taps4<RB, CELL> t0, t1, t2, t3;
                        t0.load(rt[0] + xo[0]); t1.load(rt[0] + xo[SR - 1]); t2.load(rt[SR - 1] + xo[0]); t3.load(rt[SR - 1] + xo[SR - 1]);
                        sample_acc<RB, CELL>(t0, hh[0], ll[0], xh[0], xl[0], acc_lo, acc_hi);                  // the reference's order: iy outer, ix inner
                        sample_acc<RB, CELL>(t1, hh[0], ll[0], xh[SR - 1], xl[SR - 1], acc_lo, acc_hi);
                        sample_acc<RB, CELL>(t2, hh[SR - 1], ll[SR - 1], xh[0], xl[0], acc_lo, acc_hi);
                        sample_acc<RB, CELL>(t3, hh[SR - 1], ll[SR - 1], xh[SR - 1], xl[SR - 1], acc_lo, acc_hi);
                    } else {
                        if (smask & 1u) { Taps4<RB, CELL> t; t.load(rt[0] + xo[0]); sample_acc<RB, CELL>(t, hh[0], ll[0], xh[0], xl[0], acc_lo, acc_hi); }
                        if (smask & 2u) { Taps4<RB, CELL> t; t.load(rt[0] + xo[SR - 1]); sample_acc<RB, CELL>(t, hh[0], ll[0], xh[SR - 1], xl[SR - 1], acc_lo, acc_hi); }
                        if (smask & 4u) { Taps4<RB, CELL> t; t.load(rt[SR - 1] + xo[0]); sample_acc<RB, CELL>(t, hh[SR - 1], ll[SR - 1], xh[0], xl[0], acc_lo, acc_hi); }
                        if (smask & 8u) { Taps4<RB, CELL> t; t.load(rt[SR - 1] + xo[SR - 1]); sample_acc<RB, CELL>(t, hh[SR - 1], ll[SR - 1], xh[SR - 1], xl[SR - 1], acc_lo, acc_hi); }
                    }
                    acc_lo = mul2(acc_lo, inv2); acc_hi = mul2(acc_hi, inv2);          // count 1 / 4: exact
                    float v0, v1, v2, v3;
                    unpack2f(acc_lo, v0, v1); unpack2f(acc_hi, v2, v3);
                    float* o = obase + 4 * pass;
                    const int cleft = a.C - cq;                   // channels cq .. cq + 3 are real iff index < cleft
                    if (!red) {
                        if (cleft >= 4) {
                            o[0] = v0; o[(size_t)bins] = v1; o[(size_t)2 * bins] = v2; o[(size_t)3 * bins] = v3;
                        } else {
                            if (cleft > 0) o[0] = v0;
                            if (cleft > 1) o[(size_t)bins] = v1;
                            if (cleft > 2) o[(size_t)2 * bins] = v2;
                        }
                    } else {
                        if (cleft > 0) atomicAdd(o, v0);
                        if (cleft > 1) atomicAdd(o + (size_t)bins, v1);
                        if (cleft > 2) atomicAdd(o + (size_t)2 * bins, v2);
                        if (cleft > 3) atomicAdd(o + (size_t)3 * bins, v3);
                    }
                }
            }
            e = e_next;
        }
        ibase += it.yhi - it.ya;
    }
    __syncwarp();
    if (lane == 0) sts_volatile(pub + 4u * warp, 0x7fffffff);       // nothing more to read
}

// ------------------------------------------------------------------------------------------------
// host: geometry, workspace, launches
// ------------------------------------------------------------------------------------------------
size_t align_up_sz(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct StripLayout {
    size_t ytab_off, xtab_off, zero_off, zero_bytes, rowptr_off, piece_off, entries_off, tmp_off, tmpcnt_off, ws_bytes;
};

bool strip_geometry(int levels, const float* const* bottoms, const int* heights, const int* widths, const float* scales,
                    const int* level_roi_begin, int N, int R, int C, int PH, int PW, int sr, int sm_count, int cell, StripGeom* g,
                    StripLayout* lay, unsigned* smem_bytes) {
    if (levels < 1 || levels > kMaxLevels) return false;
    if (sr < 1 || sr > 2 || PH * sr > kAxisMaxS || PW * sr > kAxisMaxS || PH > 31 || PW > 31) return false;
    if (N <= 0 || R <= 0 || R > 65535) return false;
    if ((long long)R * PH * PW * sr * sr >= (1LL << 28)) return false;
    for (int l = 0; l < levels; ++l)
        if (heights[l] < 2 || widths[l] < 2 || heights[l] > 65000) return false;
    const unsigned fixed = 128 + 256 + 8 * kMaxK;              // alignment slack + control words (pub[32], next[4]) + TMA barriers
    int best_sx = 0, best_wx = 0, best_k = 0;
    long best_score = -1;
    static const int kSx[3] = {32, 64, 96}, kHalo[3] = {8, 8, 16};
    for (int m = 0; m < 3; ++m) {
        const int sx = kSx[m];
        int k = (int)((kSmemBudget - fixed) / (unsigned)(sx * cell)) - 1;       // one physical slot is the mirror of slot 0
        if (k > kMaxK) k = kMaxK;
        if (k < 12) continue;
        const int wx = sx - kHalo[m];
        long score = 0;                                       // columns staged per row of every level, weighted by its rows
        for (int l = 0; l < levels; ++l) {
            int s = 1;
            while ((s - 1) * wx + sx < widths[l]) ++s;        // the last strip needs no halo
            score += (long)s * sx * heights[l];
        }
        if (best_score < 0 || score < best_score) { best_score = score; best_sx = sx; best_wx = wx; best_k = k; }
    }
    if (best_score < 0) return false;
    g->N = N; g->R = R; g->C = C; g->PH = PH; g->PW = PW; g->sr = sr;
    g->ny = PH * sr; g->nx = PW * sr;
    g->SX = best_sx; g->WX = best_wx; g->K = best_k; g->cell = cell;
    g->L = levels;
    int q = 0;
    long long keys = 0;
    for (int l = 0; l < levels; ++l) {
        StripLevel& lv = g->lv[l];
        lv.bottom = bottoms ? bottoms[l] : nullptr;
        lv.scale = scales ? scales[l] : 1.f;
        lv.H = heights[l]; lv.W = widths[l];
        int s = 1;
        while ((s - 1) * best_wx + best_sx < lv.W) ++s;
        lv.S = s;
        lv.q_base = q;
        lv.roi_begin = level_roi_begin ? level_roi_begin[l] : 0;
        lv.pad = 0;
        if (q + N * s > kMaxCols) return false;
        for (int c = 0; c < N * s; ++c) { g->colstart[q + c] = (int)keys; keys += lv.H; }
        q += N * s;
        if (keys > kMaxKeys) return false;
    }
    for (int l = levels; l < kMaxLevels; ++l) { g->lv[l] = g->lv[levels - 1]; g->lv[l].q_base = q; g->lv[l].roi_begin = R; }
    g->Q = q; g->keys = (int)keys;
    for (int c = q; c <= kMaxCols; ++c) g->colstart[c] = (int)keys;
    g->G = (C + 31) / 32;
    if (g->G < 1) g->G = 1;
    if (keys * g->G >= (1LL << 30)) return false;
    g->pieces = sm_count > 0 ? sm_count : kNumSMs;
    g->cap_r = PH * PW * sr * sr;                              // worst case: every sample its own fragment
    g->max_entries = R * g->cap_r;
    size_t off = 0;
    lay->ytab_off = off; off = align_up_sz(off + (size_t)R * g->ny * 16, 256);
    lay->xtab_off = off; off = align_up_sz(off + (size_t)R * g->nx * 16, 256);
    lay->zero_off = off; lay->zero_bytes = align_up_sz(((size_t)3 * g->keys + 4) * 4, 256); off += lay->zero_bytes;
    lay->rowptr_off = off; off = align_up_sz(off + ((size_t)g->keys + 1) * 4, 256);
    lay->piece_off = off; off = align_up_sz(off + ((size_t)g->pieces + 1) * 4, 256);
    lay->entries_off = off; off = align_up_sz(off + (size_t)g->max_entries * 8, 256);
    lay->tmp_off = off; off = align_up_sz(off + (size_t)g->max_entries * 16, 256);
    lay->tmpcnt_off = off; off = align_up_sz(off + (size_t)R * 4, 256);
    lay->ws_bytes = off;
    *smem_bytes = (unsigned)(g->K + 1) * (unsigned)(g->SX * cell) + fixed;
    return true;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = []() -> EncodeTiledFn {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
            (void)cudaGetLastError();
            return nullptr;
        }
        return (EncodeTiledFn)p;
    }();
    return fn;
}

// x-quad view of one NCHW level: dims (x % 4, n * C + c, x / 4, y), box (4, 32, SX / 4, 1).  Needs W % 4 == 0 and a 16-byte
// aligned base; the innermost start coordinate is always 0, so no tile load is ever misaligned (tools/tma_probe4.cu).
bool make_quad_map(CUtensorMap* map, const float* bottom, int N, int C, int H, int W, int SX) {
    EncodeTiledFn encode = encode_tiled_fn();
    if (!encode || (W & 3) || ((uintptr_t)bottom & 15u)) return false;
    const cuuint64_t dims[4] = {4, (cuuint64_t)N * (cuuint64_t)C, (cuuint64_t)(W / 4), (cuuint64_t)H};
    const cuuint64_t strides[3] = {(cuuint64_t)W * (cuuint64_t)H * 4, 16, (cuuint64_t)W * 4};
    const cuuint32_t box[4] = {4, 32, (cuuint32_t)(SX / 4), 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    return encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)bottom, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

void roi_align_strip_set_debug_buffer(unsigned long long* host_pinned) {
    cudaMemcpyToSymbol(g_strip_dead, &host_pinned, sizeof(host_pinned));      // [CTA][32] u64 watchdog records
}

size_t roi_align_strip_fpn_workspace_bytes(int levels, const int* heights, const int* widths, int N, int R, int PH, int PW, int sr) {
    StripGeom g;
    StripLayout lay;
    unsigned smem = 0;
    if (!strip_geometry(levels, nullptr, heights, widths, nullptr, nullptr, N, R, 32, PH, PW, sr, kNumSMs, kCellAsync, &g, &lay, &smem)) return 0;
    return lay.ws_bytes;
}

size_t roi_align_strip_workspace_bytes(int N, int R, int H, int W, int PH, int PW, int sr) {
    return roi_align_strip_fpn_workspace_bytes(1, &H, &W, N, R, PH, PW, sr);
}

// returns B200_ROI_OK when the path ran; kPathDeclined when it does not apply (caller falls back)
int roi_align_forward_strip_fpn(int levels, const float* const* bottoms, const int* heights, const int* widths, const float* scales,
                                const int* level_roi_begin, int N, int R, int C, int PH, int PW, int sr, const float* rois, float* top,
                                const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    if (workspace == nullptr || C <= 0) return kPathDeclined;
    if ((long long)N * C >= (1LL << 31) || (long long)R * C * PH * PW >= (1LL << 31)) return kPathDeclined;
    int sm_count = 0;
    if (device_sm_count(&sm_count) != B200_ROI_OK) return kPathDeclined;
    StripGeom g;
    StripLayout lay;
    unsigned smem = 0;
    // rows by TMA when every level has an x-quad view (W % 4 == 0, 16-byte aligned base) -- else cp.async producers
    bool tma = encode_tiled_fn() != nullptr;
    for (int l = 0; tma && l < levels; ++l) tma = (widths[l] & 3) == 0 && ((uintptr_t)bottoms[l] & 15u) == 0;
    if (!strip_geometry(levels, bottoms, heights, widths, scales, level_roi_begin, N, R, C, PH, PW, sr, sm_count,
                        tma ? kCellTma : kCellAsync, &g, &lay, &smem)) return kPathDeclined;
    if (workspace_bytes < lay.ws_bytes) return kPathDeclined;
    unsigned char* wsb = (unsigned char*)workspace;
    StripWs ws;
    ws.ytab = (uint4*)(wsb + lay.ytab_off);
    ws.xtab = (uint4*)(wsb + lay.xtab_off);
    int* zero = (int*)(wsb + lay.zero_off);
    ws.hist = zero; ws.cost = zero + g.keys; ws.maxend = zero + 2 * (size_t)g.keys;
    ws.ticket = zero + 3 * (size_t)g.keys;
    ws.rowptr = (int*)(wsb + lay.rowptr_off);
    ws.piece_start = (int*)(wsb + lay.piece_off);
    ws.entries = (uint2*)(wsb + lay.entries_off);
    ws.tmp = (uint4*)(wsb + lay.tmp_off);
    ws.tmpcnt = (int*)(wsb + lay.tmpcnt_off);

    const int xo = g.SX / 8;
    const auto prep = sr == 1 ? strip_prep<1> : strip_prep<2>;
    const auto fwd =
        tma ? (sr == 1 ? (xo == 4 ? roi_align_strip_fwd<1, 4, kCellTma> : xo == 8 ? roi_align_strip_fwd<1, 8, kCellTma> : roi_align_strip_fwd<1, 12, kCellTma>)
                       : (xo == 4 ? roi_align_strip_fwd<2, 4, kCellTma> : xo == 8 ? roi_align_strip_fwd<2, 8, kCellTma> : roi_align_strip_fwd<2, 12, kCellTma>))
            : (sr == 1 ? (xo == 4 ? roi_align_strip_fwd<1, 4, kCellAsync> : xo == 8 ? roi_align_strip_fwd<1, 8, kCellAsync> : roi_align_strip_fwd<1, 12, kCellAsync>)
                       : (xo == 4 ? roi_align_strip_fwd<2, 4, kCellAsync> : xo == 8 ? roi_align_strip_fwd<2, 8, kCellAsync> : roi_align_strip_fwd<2, 12, kCellAsync>));
    if (smem_opt_in(prep, kPrepSmemMax) != B200_ROI_OK || smem_opt_in(fwd, kSmemBudget) != B200_ROI_OK) return kPathDeclined;
    // prepass grid: one CTA per RoI when they are all resident at once (the kernel has a grid barrier), else a resident grid
    const size_t prep_dyn = (size_t)2 * (g.keys + 1) * 4 + (size_t)g.cap_r * 12;
    int per_sm = 0;
    cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, prep, kPrepThreads, prep_dyn);
    if (err != cudaSuccess || per_sm < 1) { (void)cudaGetLastError(); return kPathDeclined; }
    long long cap = (long long)per_sm * sm_count;
    const int prep_grid = (int)(R < cap ? R : cap);

    err = cudaMemsetAsync(zero, 0, lay.zero_bytes, stream);
    if (err != cudaSuccess) return (int)err;
    prep<<<prep_grid, kPrepThreads, prep_dyn, stream>>>(rois, g, ws, top, row_map);

    StripArgs a;
    a.ytab = ws.ytab; a.xtab = ws.xtab; a.entries = ws.entries; a.rowptr = ws.rowptr; a.maxend = ws.maxend;
    a.piece_start = ws.piece_start; a.out = top; a.row_map = row_map;
    a.C = C; a.G = g.G; a.K = g.K; a.WX = g.WX; a.PH = PH; a.PW = PW; a.ny = g.ny; a.nx = g.nx; a.L = g.L; a.Q = g.Q;
    a.magicK = 0xffffffffu / (unsigned)g.K + 1u;
    StripMaps maps;
    memset(&maps, 0, sizeof(maps));
    for (int l = 0; tma && l < levels; ++l)
        if (!make_quad_map(&maps.m[l], bottoms[l], N, C, heights[l], widths[l], g.SX)) return kPathDeclined;      // (the geometry was sized for TMA cells)
    a.tma = tma ? 1 : 0;
    for (int l = 0; l < kMaxLevels; ++l) a.lv[l] = g.lv[l];
    for (int c = 0; c <= kMaxCols; ++c) a.colstart[c] = g.colstart[c];

    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)g.pieces);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    err = cudaLaunchKernelEx(&cfg, fwd, maps, a);
    if (err != cudaSuccess) return (int)err;
    return finish_launch(2);
}

int roi_align_forward_strip(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                            const float* rois, float* top, const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    const int begin[2] = {0, R};
    return roi_align_forward_strip_fpn(1, &bottom, &H, &W, &scale, begin, N, R, C, PH, PW, sr, rois, top, row_map, workspace,
                                       workspace_bytes, stream);
}

}  // namespace b200
