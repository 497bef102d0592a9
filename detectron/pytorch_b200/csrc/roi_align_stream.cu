// roi_align_stream.cu -- Caffe2-exact RoIAlign FORWARD, "streaming strip" fast path (cp.async + mbarrier ring).
//
// The feature map is cut into vertical strips of WX columns (+ a halo); one persistent CTA per SM owns a
// contiguous piece of the linear space (image, strip, 32-channel group, row) and streams the rows of its
// strips top to bottom through a ring of K row slots in shared memory.  Four producer warps fetch rows with
// 4-byte cp.async (LDGSTS: global -> shared without a register round trip, 128-byte coalesced per warp) and
// signal per-slot mbarriers (cp.async.mbarrier.arrive); they run ahead of 16 consumer warps, which release
// slots on a second set of mbarriers, so loading overlaps the arithmetic completely.
//
// Shared-memory layout of one row slot: [32 channels][SX columns], SX odd.  The compute mapping is
// lane = channel: one warp evaluates one bilinear tap of one sample for 32 channels with ONE conflict-free
// LDS.32 (bank = c * SX + x), and all addressing / weights are warp-uniform.
// Why not TMA (cp.async.bulk.tensor): skewed channel rows would need tile loads at unaligned innermost start
// coordinates, and with TMA's 16-byte placement granularity every channel row would start at a bank that is a multiple of 4 -- a lane = channel access would hit at most 8 banks (4-way conflict).
// The 4-byte cp.async can place a row at any word, which is what the odd channel stride needs.
//
// Work = "fragments": up to 8 consecutive bins of one bin row of one RoI, keyed by the first feature row
// they read.  A fragment is processed by ONE warp when the rows [key, end) it needs are resident, so every
// output element is computed by one lane in the reference's own operation order: bit-identical to the
// reference kernel, deterministic, no zero-fill of the output.  Only bins whose samples cannot be resident
// together (x-span beyond the strip halo, y-span beyond the ring) are cut into per-sample fragments that
// accumulate with red.global.add onto elements the prepass zeroed (at most two partial sums per element ->
// still deterministic).
//
// Output: staged once, transposed once.  The bin loop stores each bin's result for lane = channel into its own
// output row laid out (bin, channel): one aligned 128-byte line per bin and 32-channel group.  (The (channel, bin)
// layout would give every store a run of at most 8 floats inside one channel plane -- part of a 32-byte sector,
// and such a store that misses L2 stalls the memory pipeline the bin loop's shared-memory loads share.)  After
// a grid barrier every CTA transposes whole rows in place to (channel, bin) through shared memory.
//
// Prepass (channel independent): `clear` zeroes the counters; `prep`, ONE kernel launched as its programmatic
// dependent, builds the per-RoI axis tables (all IEEE divisions; ring-slot byte offsets precomputed), lists the
// fragments and takes each one's rank within its (image, strip, row) key with a returning atomic, passes a grid
// barrier, scans the histogram in every CTA's shared memory (CSR row pointers), writes the 8-byte fragment records
// at row pointer + rank and cuts the linear space into one piece per SM of equal estimated cost.  The main kernel
// is launched as the prepass's programmatic dependent: its ring and barrier set-up overlaps the prepass.
//
// Semantics: lib/modeling/roi_xfrom/roi_align/src/roi_align_kernel.cu (reference) :16-63, :65-121.
#include "common.cuh"
#include "strip_prep.cuh"
#include <type_traits>
#include <string.h>
#include <stdlib.h>

namespace b200 {

namespace {

constexpr int kConsumerWarps = 16;
constexpr int kProducerWarps = 4;
constexpr int kStreamThreads = 32 * (kConsumerWarps + kProducerWarps);
constexpr int kFragBins = 8;                                  // bins per fragment
constexpr int kTabWords = 18 * 4;                              // per-warp axis-table buffer: 16 x entries + 2 y entries
constexpr int kMaxSlots = 32;                                 // ring depth K <= 32 (phase bits live in one register)
constexpr unsigned kBarBytes = 2 * kMaxSlots * 8;             // full[] and empty[] mbarriers, at the start of dynamic shared memory
constexpr int kAxisMaxS = 32;                                 // P * sampling_ratio per axis
constexpr int kPrepThreads = 128;
constexpr unsigned kRowCost = 8u;                             // cost of streaming one row (16 acquires + staging), in bins
constexpr unsigned kSmemBudget = 227u * 1024u;
constexpr unsigned kPrepSmemMax = 200u * 1024u;               // dynamic shared memory of the prepass: scan of the keys + one RoI's fragment list

typedef unsigned long long u64;

constexpr int kMaxLevels = 6;                                 // feature maps served by one launch (FPN: P2..P6)
constexpr int kMaxCols = 96;                                  // strip columns (level, image, strip) of one launch

struct StreamLevel {                                          // one feature map of the pyramid (a plain call has one)
    const float* bottom;                                      // (N, C, H, W)
    float scale;
    int H, W, S;                                              // S: strips per image
    int q_base;                                               // its first strip column; column = q_base + image * S + strip
    int roi_begin;                                            // its first RoI (RoIs are stored level-major)
    int pad;
};

struct StreamGeom {
    int N, R, C, PH, PW, sr;
    int ny, nx;
    int SX, WX, K;              // columns held per row (odd, 32 m + 1), strip core width, ring depth
    int row_bytes;              // bytes of one ring slot = 32 * SX * 4
    int L;                      // levels
    int Q, keys;                // strip columns, keys = sum over columns of their rows
    int G;                      // 32-channel groups
    int pieces;                 // persistent CTAs
    int max_entries, cap_r;     // cap_r: fragments one RoI can have at most
    int tail_rows;              // output rows the main kernel's tail holds in shared memory at once
    StreamLevel lv[kMaxLevels];
    int colstart[kMaxCols + 1]; // first key of every column (its rows are consecutive keys); colstart[Q] = keys
};

// level of RoI r / of strip column q (at most kMaxLevels entries: linear scan)
__host__ __device__ __forceinline__ int level_of_roi(const StreamGeom& g, int r) {
    int l = 0;
    while (l + 1 < g.L && r >= g.lv[l + 1].roi_begin) ++l;
    return l;
}

struct StreamWs {
    uint4* ytab;                // [R][ny] {hy, ly, byte offset of the ring slot of row y_low, 0}; the lower tap row is the NEXT slot
    uint4* xtab;                // [R][nx] {hx, lx, x_low * 4, 0}
    int* hist;                  // [keys] fragments per key                           (zero block)
    int* cost;                  // [keys] estimated cost per key                      (zero block)
    int* maxend;                // [keys] max over the key's fragments of `end`       (zero block)
    int* ticket;                // [4] grid barriers: [0] the prepass's, [1] the main kernel's (zero block)
    int* rowptr;                // [keys + 1] CSR offsets into entries
    int* piece_start;           // [pieces + 1] linear start index of every piece
    uint2* entries;             // fragment records
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

// ------------------------------------------------------------------------------------------------
// axis samples, adjusted so that both taps are always inside the map
// ------------------------------------------------------------------------------------------------
struct AdjTap {
    int   low;                  // low cell in [0, size - 2]
    float l, h;                 // weights of cell low + 1 / cell low (0, 0 for a sample the reference skips)
};

// The reference clamps a sample on the last cell to low = high = size - 1 with weights (h, l) = (1, 0).  Reading
// cells (size - 2, size - 1) with weights (0, 1) instead is the same sum term for term (x*1 and y*0 swap places in
// the FMA chain; the zero products do not change any finite partial sum), and keeps every tap in the map.
__device__ __forceinline__ AdjTap adj_axis(float v, int size) {
    const AxisTap t = xfrom_axis(v, size);
    AdjTap a;
    a.low = t.low; a.l = t.l; a.h = t.h;
    if (t.low >= size - 1) { a.low = size - 2; a.l = 1.f; a.h = 0.f; }
    if (!t.valid) { a.l = 0.f; a.h = 0.f; }
    return a;
}

// Enumerate the fragments of bin row `ph` of one RoI.  yl / yh: the reference's low / high tap row per y sample
// (equal on the clamped last row); xl: adjusted low cell per x sample.
// emit(strip, key, end, pw0, npw, smask, red, zero_owner)
template <int SR, class Emit>
__device__ __forceinline__ void enum_row(const int* yl, const int* yh, const int* xl, int ph, const StreamGeom& g, int S, Emit&& emit) {
    const int i0 = ph * SR, i1 = i0 + SR - 1;
    int ngroups = 1;
    int key[2], end[2];
    unsigned ym[2];
    key[0] = yl[i0]; end[0] = yh[i1] + 1; ym[0] = (1u << SR) - 1u;
    key[1] = 0; end[1] = 0; ym[1] = 0;
    if (SR == 2 && end[0] - key[0] > g.K) {          // rows cannot be resident together: one fragment per y sample
        ngroups = 2;
        end[0] = yh[i0] + 1; ym[0] = 1u;
        key[1] = yl[i1]; end[1] = yh[i1] + 1; ym[1] = 2u;
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
// prepass: clear of the counters, then ONE kernel: tables + fragment list | grid barrier | CSR scan (every CTA) | records,
// zero-fill, pieces
// ------------------------------------------------------------------------------------------------
// The counters the prepass accumulates into must start at zero.  A kernel instead of a memset: the prepass is launched as
// its programmatic dependent, so that its tables and fragment lists are computed while this runs.
__global__ void __launch_bounds__(kPrepThreads)
stream_clear(int4* __restrict__ zero, int n16) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    for (int i = blockIdx.x * kPrepThreads + threadIdx.x; i < n16; i += gridDim.x * kPrepThreads) zero[i] = make_int4(0, 0, 0, 0);
}

template <int SR>
__global__ void __launch_bounds__(kPrepThreads)
stream_prep(const float* __restrict__ rois, StreamGeom g, StreamWs ws, float* __restrict__ out, const int* __restrict__ row_map) {
    extern __shared__ unsigned s_dyn[];                       // [keys + 1] fragment prefix, [keys + 1] cost prefix, [cap_r][3] fragment list
    __shared__ int s_nlist;
    __shared__ int s_yl[kAxisMaxS], s_yh[kAxisMaxS], s_xl[kAxisMaxS];
    __shared__ unsigned short s_zero[kAxisMaxS * kAxisMaxS];
    __shared__ int s_nzero;
    __shared__ unsigned s_ph[kPrepThreads], s_pc[kPrepThreads];
    const int t = threadIdx.x;
    const int keys = g.keys;
    unsigned* s_pre = s_dyn;
    unsigned* s_cpre = s_dyn + (keys + 1);
    unsigned* s_list = s_dyn + 2 * (keys + 1);               // {key index, record.x, record.y} per fragment of the current RoI
    // the main kernel may start its prologue (ring, barriers) on every SM this grid leaves room on; it waits for all of
    // this grid's results before it reads any of them
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

    // ---- phase 1: per RoI (the grid loops over them when R exceeds the resident grid): axis tables (all IEEE divisions live
    // here), the fragments listed in shared memory by the bin-row threads; then ALL threads take one fragment each: rank
    // within its key (one returning atomic, its latency hides behind the grid barrier), cost / extent atomics, and a
    // temporary record that phase 3 only has to drop into the CSR
    for (int r = blockIdx.x; r < g.R; r += gridDim.x) {
        __syncthreads();                                      // s_yl / s_yh / s_xl / s_list of the previous RoI are no longer read
        const StreamLevel& lv = g.lv[level_of_roi(g, r)];
        const XfromRoi geo = xfrom_roi(rois + 5 * (size_t)r, lv.scale, g.PH, g.PW, g.sr);
        if (t == 0) s_nlist = 0;
        if (t < g.ny + g.nx) {
            const bool isy = t < g.ny;
            const int s = isy ? t : t - g.ny;
            if (isy) {
                // rows exactly as the reference takes them (low == high == H - 1 on the clamped last row, weights (1, 0)): the
                // lower tap then reads whatever the next ring slot holds with weight 0 -- always finite, the ring starts zeroed
                const AxisTap a = xfrom_axis(xfrom_coord(geo.start_h, geo.bin_h, s / SR, s % SR, SR), lv.H);
                s_yl[s] = a.low; s_yh[s] = a.high;
                uint4 e;
                e.x = __float_as_uint(a.valid ? a.h : 0.f); e.y = __float_as_uint(a.valid ? a.l : 0.f);
                e.z = (unsigned)((a.low % g.K) * g.row_bytes);
                e.w = 0u;
                ws.ytab[(size_t)r * g.ny + s] = e;
            } else {
                const AdjTap a = adj_axis(xfrom_coord(geo.start_w, geo.bin_w, s / SR, s % SR, SR), lv.W);
                s_xl[s] = a.low;
                uint4 e;
                e.x = __float_as_uint(a.h); e.y = __float_as_uint(a.l);
                e.z = (unsigned)(a.low * 4); e.w = 0u;
                ws.xtab[(size_t)r * g.nx + s] = e;
            }
        }
        __syncthreads();
        const bool batch_ok = geo.batch >= 0 && geo.batch < g.N;
        if (batch_ok && t < g.PH) {
            const int cbase = lv.q_base + geo.batch * lv.S;
            enum_row<SR>(s_yl, s_yh, s_xl, t, g, lv.S, [&](int s, int key, int end, int pw0, int npw, unsigned smask, int red, bool owner) {
                const int idx = atomicAdd(&s_nlist, 1);
                const uint2 e = pack_entry(r, t, pw0, npw, red, key, end, smask);
                s_list[3 * idx] = (unsigned)(g.colstart[cbase + s] + key); s_list[3 * idx + 1] = e.x; s_list[3 * idx + 2] = e.y;
                (void)owner;
            });
        }
        __syncthreads();
        // the counters are cleared by the kernel this one depends on: wait for it before the first atomic (returns at once
        // from the second RoI on)
        asm volatile("griddepcontrol.wait;" ::: "memory");
        const int n = s_nlist;
        for (int idx = t; idx < n; idx += kPrepThreads) {
            const unsigned k = s_list[3 * idx], ex = s_list[3 * idx + 1], ey = s_list[3 * idx + 2];
            const int npw = (int)((ex >> 26) & 7u) + 1, end = (int)(ey & 0xffffu) + (int)((ey >> 16) & 0xffu);
            const int rank = atomicAdd(&ws.hist[k], 1);
            atomicAdd(&ws.cost[k], 2 + npw);
            atomicMax(&ws.maxend[k], end);
            ws.tmp[(size_t)r * g.cap_r + idx] = make_uint4(k, (unsigned)rank, ex, ey);
        }
        if (t == 0) ws.tmpcnt[r] = batch_ok ? n : -1;
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");      // a CTA without a RoI still arrives on a cleared ticket
    // ---- grid barrier (the grid is sized to be resident: see the launcher)
    prepass::grid_barrier(ws.ticket);
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
        if (nz > 0) {                                         // the output row is in the main kernel's staging layout (bin, channel)
            float* out_r = out + (size_t)(row_map ? row_map[r] : r) * g.C * bins;
            for (int idx = t; idx < g.C * nz; idx += kPrepThreads) {
                const int k = idx / g.C, c = idx - k * g.C;
                out_r[(size_t)s_zero[k] * g.C + c] = 0.f;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// PTX helpers: mbarrier + cp.async
// ------------------------------------------------------------------------------------------------
// Watchdog evidence: a wait that is half way to the trap leaves a record here ([CTA][32] u64; host-pinned, optional).
__device__ u64* g_stream_dead = nullptr;

__device__ __forceinline__ unsigned smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned bar, unsigned parity) {
    unsigned ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"     // %3: the hardware may park the thread this long (ns)
        "selp.u32 %0, 1, 0, p;\n"
        "}" : "=r"(ok) : "r"(bar), "r"(parity), "r"(20000u) : "memory");
    return ok != 0;
}
// try_wait suspends the thread in hardware for a bounded time per attempt.  A wait that is still pending after 2^20
// attempts (seconds) is a protocol bug: trap (surfaces as a launch failure) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity, unsigned tag = 0u) {
    if (mbar_try_wait(bar, parity)) return;
    int spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        ++spins;
        if (spins == (1 << 19) && g_stream_dead != nullptr && (threadIdx.x & 31) == 0) {
            // half way to the trap: say who is stuck on what (host-pinned buffer registered by the caller, else nothing)
            g_stream_dead[blockIdx.x * 32 + (threadIdx.x >> 5)] =
                0xDEAD000000000000ull | ((u64)tag << 16) | ((u64)parity << 8) | (u64)((bar >> 3) & 0xff);
            __threadfence_system();
        }
        if (spins > (1 << 20)) __trap();
    }
}
// L2 eviction priorities.  Each feature row is read once (evict_first); the staged output rows are read back by the tail, so
// they are kept (evict_last) until the tail rewrites them (evict_normal, which also leaves no evict_last lines behind).
// At cfg2 the staged rows are 26 MB of the 50 MB L2 while 56 MB of features stream through it.
__device__ __forceinline__ u64 l2_evict_first() { u64 p; asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ u64 l2_evict_last() { u64 p; asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ u64 l2_evict_normal() { u64 p; asm("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ void st_hint(float* p, float v, u64 pol) {
    asm volatile("st.global.L2::cache_hint.f32 [%0], %1, %2;" ::"l"(p), "f"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint(float* p, float4 v, u64 pol) {
    asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}
// 4-byte cp.async (LDGSTS): global -> shared without registers.
__device__ __forceinline__ void cp_async4(unsigned dst, const float* src, u64 pol) {
    asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "l"(pol) : "memory");
}
// ok == false copies nothing and zero-fills the word
__device__ __forceinline__ void cp_async4_if(unsigned dst, const float* src, bool ok, u64 pol) {
    asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 4, %2, %3;" ::"r"(dst), "l"(src), "r"(ok ? 4 : 0), "l"(pol) : "memory");
}
// the mbarrier receives one arrival from this thread once all its earlier cp.async have landed
__device__ __forceinline__ void cp_async_arrive(unsigned bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ uint4 lds128(unsigned addr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}

struct StreamArgs {
    const uint4* ytab;
    const uint4* xtab;
    const uint2* entries;
    const int* rowptr;
    const int* maxend;
    const int* piece_start;
    float* out;
    const int* row_map;
    int* ticket;                // grid barrier between the fragments and the transpose (zeroed by stream_clear)
    int R, C, G, K, WX, PH, PW, ny, nx, L, Q;
    int tail_rows;
    StreamLevel lv[kMaxLevels];
    int colstart[kMaxCols + 1];
};

// one item = the part of one (strip column q, channel group) that lies in this CTA's piece
struct Item {
    int lvl, n, s, g, ya, yb, e0, e1, yhi, kbase;
};

// Decode the item that starts at linear index L (all lanes of the calling warp; yhi by warp reduction).
__device__ __forceinline__ Item decode_item(int L, int L1, const StreamArgs& a, int lane) {
    Item it;
    int lo = 0, hi = a.Q - 1;                                  // column: the last one whose first linear index is <= L
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
    it.e0 = __ldcg(&a.rowptr[it.kbase + it.ya]);
    it.e1 = __ldcg(&a.rowptr[it.kbase + it.yb]);
    int m = 0;
    if (it.e1 > it.e0) {
        for (int y = it.ya + lane; y < it.yb; y += 32) m = max(m, __ldcg(&a.maxend[it.kbase + y]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    }
    it.yhi = m;
    return it;
}

// fp32 pairs in one 64-bit register pair, used for the warp-uniform weight products.  sm_90 has no packed fp32x2
// multiply: two __fmul_rn, one per half.
__device__ __forceinline__ u64 pack2f(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void unpack2f(u64 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ u64 mul2f(u64 a, u64 b) {
    float a0, a1, b0, b1; unpack2f(a, a0, a1); unpack2f(b, b0, b1);
    return pack2f(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}

struct Taps { float v1, v2, v3, v4; };

// The four taps of one sample for this lane's channel: rows (slot, slot + 1) x columns (x_low, x_low + 1).  The lower row
// always sits in the NEXT physical slot (the ring has a mirror of slot 0 behind slot K - 1), so one address serves all four.
template <int RB>
__device__ __forceinline__ Taps load_taps(unsigned at) {
    Taps t;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(t.v1) : "r"(at));
    asm volatile("ld.shared.f32 %0, [%1+4];" : "=f"(t.v2) : "r"(at));
    asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(t.v3) : "r"(at), "n"(RB));
    asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(t.v4) : "r"(at), "n"(RB + 4));
    return t;
}

// One bilinear sample, the reference's rounding recipe:
// val = FFMA(v4, w4, FFMA(v3, w3, FFMA(v1, w1, FMUL(v2, w2)))) with w1 = hy*hx, w2 = hy*lx, w3 = ly*hx, w4 = ly*lx.
// hyhy = (hy, hy), lyly = (ly, ly), hxlx = (hx, lx) packed.
__device__ __forceinline__ float sample_val(const Taps& t, u64 hyhy, u64 lyly, u64 hxlx) {
    float w1, w2, w3, w4;
    unpack2f(mul2f(hyhy, hxlx), w1, w2);
    unpack2f(mul2f(lyly, hxlx), w3, w4);
    return __fmaf_rn(t.v4, w4, __fmaf_rn(t.v3, w3, __fmaf_rn(t.v1, w1, __fmul_rn(t.v2, w2))));
}

// Stage row y of one (image, strip, channel group) into a ring slot: M full 32-column chunks per channel
// (lane = column: 128-byte coalesced) plus the last column x = 32 M for all channels at once (lane = channel),
// with 4-byte cp.async.
template <int M>
__device__ __forceinline__ void stage_row(const float* __restrict__ src_row, size_t plane, unsigned dst, int xw, int cvalid, int lane) {
    const u64 pol = l2_evict_first();
    // src_row: (channel 0, row y, column x0); xw = number of valid columns from x0; cvalid = number of real channels
    constexpr int SX = 32 * M + 1;
    if (cvalid == 32 && xw >= SX) {                           // interior: no predicates, constant offsets
        const float* sc = src_row + lane;
        const unsigned d = dst + (unsigned)lane * 4u;
#pragma unroll 8
        for (int c = 0; c < 32; ++c) {
#pragma unroll
            for (int m = 0; m < M; ++m) cp_async4(d + (unsigned)(c * SX + 32 * m) * 4u, sc + 32 * m, pol);
            sc += plane;
        }
        cp_async4(dst + (unsigned)(lane * SX + 32 * M) * 4u, src_row + (size_t)lane * plane + 32 * M, pol);
    } else {
#pragma unroll 4
        for (int c = 0; c < 32; ++c) {
            const bool cok = c < cvalid;
            const float* sc = src_row + (size_t)(cok ? c : 0) * plane;
#pragma unroll
            for (int m = 0; m < M; ++m) {
                const int x = lane + 32 * m;
                const bool ok = cok && x < xw;
                cp_async4_if(dst + (unsigned)(c * SX + x) * 4u, sc + (ok ? x : 0), ok, pol);
            }
        }
        const bool ok = lane < cvalid && 32 * M < xw;
        cp_async4_if(dst + (unsigned)(lane * SX + 32 * M) * 4u, src_row + (ok ? (size_t)lane * plane + 32 * M : 0), ok, pol);
    }
}

// The CTA's piece [L0, L1) of the linear space: producers stream its rows through the ring, consumers compute its fragments
// and store every bin's result into the output row's staging layout (bin, channel).  ring: K + 1 slots of RB bytes, then
// kConsumerWarps per-warp axis-table buffers of kTabWords words.
template <int SR, int M>
__device__ __forceinline__ void stream_fragments(const StreamArgs& a, unsigned ring, unsigned bars, int L0, int L1) {
    constexpr int SX = 32 * M + 1;
    constexpr int RB = 128 * SX;                                  // bytes of one ring slot
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    if (warp >= kConsumerWarps) {
        // =============================== producers ===============================
        // Row i of the CTA's row stream (all items, in order) is staged by producer warp i % kProducerWarps.  Every
        // producer tracks the phase of every slot (one flip per row of the stream) but waits only for its own rows.
        const int pw = warp - kConsumerWarps;
        unsigned ephase = 0xffffffffu;                // waiting for parity 1 on a fresh barrier passes immediately
        int turn = 0;                                 // stream row index modulo kProducerWarps
        for (int L = L0; L < L1;) {
            const Item it = decode_item(L, L1, a, lane);
            L += it.yb - it.ya;
            if (it.e1 <= it.e0) continue;
            int slot = it.ya % a.K;
            const StreamLevel& lv = a.lv[it.lvl];
            const size_t plane = (size_t)lv.H * lv.W;
            const int x0 = it.s * a.WX;
            const int c0 = it.g * 32;
            const int cvalid = min(32, a.C - c0);
            const int xw = lv.W - x0;
            const int rowlen = lv.W;
            const float* src = lv.bottom + ((size_t)it.n * a.C + c0) * plane + (size_t)it.ya * lv.W + x0;
            for (int y = it.ya; y < it.yhi; ++y) {
                // EVERY producer waits for EVERY row's slot, not only for the rows it stages: successive uses of a slot can
                // belong to different producer warps (K % kProducerWarps != 0, or an item boundary), and a parity wait that
                // runs two phases ahead of its barrier passes at once -- a producer that skipped the wait of use k - 1 could
                // overtake the warp that stages it and overwrite use k - 2.  Having seen use k - 2 released here, the test
                // for use k can only be one phase ahead (measured: K = 15, four producers, rows 2 and 17 of one item).
                const unsigned full = bars + 8u * slot, empty = bars + 8u * (kMaxSlots + slot);
                mbar_wait(empty, (ephase >> slot) & 1u, 0x1000u + (unsigned)y);
                if (turn == pw) {
                    stage_row<M>(src, plane, ring + (unsigned)slot * (unsigned)RB, xw, cvalid, lane);
                    if (slot == 0) stage_row<M>(src, plane, ring + (unsigned)a.K * (unsigned)RB, xw, cvalid, lane);   // mirror
                    cp_async_arrive(full);
                }
                ephase ^= 1u << slot;
                if (++slot == a.K) slot = 0;
                if (++turn == kProducerWarps) turn = 0;
                src += rowlen;
            }
        }
        return;
    }

    // =============================== consumers ===============================
    const unsigned tbuf = ring + (unsigned)(a.K + 1) * (unsigned)RB + (unsigned)(warp * kTabWords) * 4u;   // 16-byte aligned
    const unsigned lane_base = ring + (unsigned)(lane * SX) * 4u;
    const int bins = a.PH * a.PW;
    unsigned fphase = 0u;
    constexpr float kInvCount = 1.f / (float)(SR * SR);
    const u64 keep = l2_evict_last();                             // the tail reads the staged rows back

    for (int L = L0; L < L1;) {
        const Item it = decode_item(L, L1, a, lane);
        L += it.yb - it.ya;
        if (it.e1 <= it.e0) continue;
        const unsigned lc = lane_base - (unsigned)(it.s * a.WX) * 4u;
        int acq = it.ya, rel = it.ya;
        int acq_slot = it.ya % a.K, rel_slot = acq_slot;
        const int c0 = it.g * 32;
        const bool cok = c0 + lane < a.C;
        // every warp waits for every row of the item before it releases it, in stream order (keeps the per-slot
        // phase bits in step with the producers)
        auto acquire_to = [&](int row_end, unsigned tag) {
            while (acq < row_end) {
                mbar_wait(bars + 8u * acq_slot, (fphase >> acq_slot) & 1u, tag + (unsigned)acq);
                fphase ^= 1u << acq_slot;
                ++acq;
                if (++acq_slot == a.K) acq_slot = 0;
            }
        };
        auto release_to = [&](int row_end) {                  // rows [rel, row_end) have been acquired
            if (rel < row_end) {
                if (lane == 0) {
                    int rs = rel_slot;
                    for (int y = rel; y < row_end; ++y) { mbar_arrive(bars + 8u * (kMaxSlots + rs)); if (++rs == a.K) rs = 0; }
                }
                rel_slot += row_end - rel;                     // one wrap at most in the common case: no division
                while (rel_slot >= a.K) rel_slot -= a.K;
                rel = row_end;
            }
        };

        // Fragment pipeline (global-load latency is the enemy: entries and tables are needed by every lane at once):
        //   entry records are fetched two fragments ahead; the axis tables of the NEXT fragment are fetched one fragment
        //   ahead, lane-distributed (lanes 0..15: its x entries, lanes 16..17: its y entries -- one 16-byte load per lane),
        //   parked in registers, and dropped into this warp's table buffer in shared memory when their fragment starts;
        //   the bin loop then reads them with broadcast LDS.128.
        auto load_tab = [&](const uint2& en) -> uint4 {
            const int rn = en.x & 0xffffu, phn = (en.x >> 16) & 31u, pwn = (en.x >> 21) & 31u, nn = (int)((en.x >> 26) & 7u) + 1;
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            const bool isx = lane < nn * SR;                   // one predicated load: the two tables differ in base and index only
            const uint4* base = isx ? a.xtab : a.ytab;
            const int idx = isx ? rn * a.nx + pwn * SR + lane : rn * a.ny + phn * SR + (lane - 16);
            if (isx || (lane >= 16 && lane < 16 + SR)) v = __ldcg(base + idx);
            return v;
        };
        int e = it.e0 + warp;
        uint2 ent0 = make_uint2(0u, 0u), ent1 = make_uint2(0u, 0u);
        uint4 tab = make_uint4(0u, 0u, 0u, 0u);
        if (e < it.e1) { ent0 = __ldcg(&a.entries[e]); tab = load_tab(ent0); }
        if (e + kConsumerWarps < it.e1) ent1 = __ldcg(&a.entries[e + kConsumerWarps]);
        while (e < it.e1) {
            const uint2 cur = ent0;
            const int e_next = e + kConsumerWarps;
            // this fragment's tables -> shared (the previous fragment's readers are past their last LDS: trailing syncwarp)
            if (lane < 18) asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(tbuf + lane * 16), "r"(tab.x), "r"(tab.y), "r"(tab.z), "r"(tab.w) : "memory");
            __syncwarp();
            ent0 = ent1;
            if (e_next < it.e1) tab = load_tab(ent0);                               // in flight while this fragment computes
            if (e_next + kConsumerWarps < it.e1) ent1 = __ldcg(&a.entries[e_next + kConsumerWarps]);
            const int r = cur.x & 0xffffu, ph = (cur.x >> 16) & 31u, pw0 = (cur.x >> 21) & 31u;
            const int npw = (int)((cur.x >> 26) & 7u) + 1;
            const bool red = (cur.x >> 29) & 1u;
            const int key = cur.y & 0xffffu, end = key + (int)((cur.y >> 16) & 0xffu);
            const unsigned smask = (cur.y >> 24) & 0xfu;
            // entries are sorted by key: rows below it are done with.  Rows this warp never needed are passed through one
            // at a time (waited for, then released at once): holding them while waiting for later rows would starve the
            // producers of slots whenever this warp's consecutive fragments lie more than K rows apart.
            release_to(min(acq, key));
            while (acq < key) {
                acquire_to(acq + 1, 0x2000u);
                release_to(acq);
            }
            const int orow = a.row_map ? __ldg(&a.row_map[r]) : r;       // lands while this warp waits for its rows
            acquire_to(end, 0x2800u);                           // rows [key, end) must be resident
            const uint4 yA = lds128(tbuf + 16 * 16);
            uint4 yB = yA;
            if (SR == 2) yB = lds128(tbuf + 17 * 16);
            // row bases for this lane and the packed axis weights (uniform; hoisted out of the bin loop)
            const unsigned rt0 = lc + yA.z, rt1 = lc + yB.z;
            const u64 hh0 = pack2f(__uint_as_float(yA.x), __uint_as_float(yA.x)), ll0 = pack2f(__uint_as_float(yA.y), __uint_as_float(yA.y));
            const u64 hh1 = pack2f(__uint_as_float(yB.x), __uint_as_float(yB.x)), ll1 = pack2f(__uint_as_float(yB.y), __uint_as_float(yB.y));
            unsigned tb = tbuf;                                   // this bin's x entries (broadcast reads)
            // this lane's result of the bin: output row orow in the staging layout (bin, channel)
            float* op = a.out + ((size_t)orow * bins + ph * a.PW + pw0) * a.C + c0 + lane;
            const unsigned tb_end = tbuf + (unsigned)npw * (SR * 16u);
            if (SR == 2 && smask == 0xfu) {
                // whole bins (the common case): all 16 taps are requested before the first one is used
                do {
                    const uint4 cxA = lds128(tb), cxB = lds128(tb + 16);
                    const u64 wxA = pack2f(__uint_as_float(cxA.x), __uint_as_float(cxA.y));
                    const u64 wxB = pack2f(__uint_as_float(cxB.x), __uint_as_float(cxB.y));
                    const Taps t0 = load_taps<RB>(rt0 + cxA.z);
                    const Taps t1 = load_taps<RB>(rt0 + cxB.z);
                    const Taps t2 = load_taps<RB>(rt1 + cxA.z);
                    const Taps t3 = load_taps<RB>(rt1 + cxB.z);
                    float acc = __fadd_rn(0.f, sample_val(t0, hh0, ll0, wxA));   // the reference's order: iy outer, ix inner
                    acc = __fadd_rn(acc, sample_val(t1, hh0, ll0, wxB));
                    acc = __fadd_rn(acc, sample_val(t2, hh1, ll1, wxA));
                    acc = __fadd_rn(acc, sample_val(t3, hh1, ll1, wxB));
                    if (cok) st_hint(op, __fmul_rn(acc, kInvCount), keep);      // count 4: exact
                    tb += 32u; op += a.C;
                } while (tb != tb_end);
            } else {
                do {
                    const uint4 cxA = lds128(tb);
                    uint4 cxB = cxA;
                    if (SR == 2) cxB = lds128(tb + 16);
                    const u64 wxA = pack2f(__uint_as_float(cxA.x), __uint_as_float(cxA.y));
                    const u64 wxB = pack2f(__uint_as_float(cxB.x), __uint_as_float(cxB.y));
                    float acc = 0.f;
                    if (SR == 1) {
                        acc = __fadd_rn(acc, sample_val(load_taps<RB>(rt0 + cxA.z), hh0, ll0, wxA));
                    } else {
                        if (smask & 1u) acc = __fadd_rn(acc, sample_val(load_taps<RB>(rt0 + cxA.z), hh0, ll0, wxA));
                        if (smask & 2u) acc = __fadd_rn(acc, sample_val(load_taps<RB>(rt0 + cxB.z), hh0, ll0, wxB));
                        if (smask & 4u) acc = __fadd_rn(acc, sample_val(load_taps<RB>(rt1 + cxA.z), hh1, ll1, wxA));
                        if (smask & 8u) acc = __fadd_rn(acc, sample_val(load_taps<RB>(rt1 + cxB.z), hh1, ll1, wxB));
                    }
                    const float v = __fmul_rn(acc, kInvCount);     // count 1 / 4: exact
                    if (cok) {
                        if (red) atomicAdd(op, v);
                        else st_hint(op, v, keep);
                    }
                    tb += SR * 16u; op += a.C;
                } while (tb != tb_end);
            }
            __syncwarp();                                       // the table buffer is rewritten for the next fragment
            e = e_next;
        }
        // item tail: nothing more to read -- give back what is held, then pass the remaining rows through one by one
        // (a warp that held rows while waiting for later ones could starve the producers of slots)
        release_to(acq);
        while (acq < it.yhi) {
            acquire_to(acq + 1, 0x3000u);
            release_to(acq);
        }
        __syncwarp();
    }
}

// Words per bin of a row block in the tail's shared memory: odd, so that the lanes of a warp that read one channel at
// consecutive bins hit distinct banks.
__host__ __device__ __forceinline__ int tail_stride(int C) { return C | 1; }

__device__ __forceinline__ void put_floats(float* d, float v) { d[0] = v; }
__device__ __forceinline__ void put_floats(float* d, float4 v) { d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w; }

// Transpose this CTA's output rows r = blockIdx.x + j * gridDim.x in place, from (bin, channel) to (channel, bin), through
// shared memory s, a.tail_rows rows at a time: every element of a batch is read before any is written, and no other CTA
// touches these rows.  V = 4: 16-byte loads and stores (C % 4 == 0 and a 16-byte aligned output); else V = 1.  The rows were
// written by other CTAs of this grid: L2 loads (.cg), never .nc (DESIGN.md 4.1).
template <int V>
__device__ __forceinline__ void transpose_rows(const StreamArgs& a, float* s) {
    using VT = typename std::conditional<V == 4, float4, float>::type;
    constexpr int kUnroll = 4;                                    // loads in flight per thread
    const int tid = threadIdx.x;
    const int C = a.C, bins = a.PH * a.PW, cs = tail_stride(C);
    const int nv = C * bins / V;                                  // V-wide items of one row
    const int* row_map = a.row_map;
    const u64 norm = l2_evict_normal();
    for (int r0 = blockIdx.x; r0 < a.R; r0 += a.tail_rows * (int)gridDim.x) {
        const int nrows = min(a.tail_rows, (a.R - r0 + (int)gridDim.x - 1) / (int)gridDim.x);
        const int n = nrows * nv;
        for (int i0 = tid; i0 < n; i0 += kUnroll * kStreamThreads) {
            VT v[kUnroll];
            int at[kUnroll];                                      // where item u goes in shared memory
#pragma unroll
            for (int u = 0; u < kUnroll; ++u) {
                const int i = i0 + u * kStreamThreads;
                if (i < n) {
                    const int j = i / nv, f = (i - j * nv) * V;
                    const int r = r0 + j * (int)gridDim.x;
                    const int orow = row_map ? row_map[r] : r;
                    v[u] = __ldcg(reinterpret_cast<const VT*>(a.out + (size_t)orow * C * bins + f));
                    const int b = f / C;
                    at[u] = (j * bins + b) * cs + (f - b * C);
                }
            }
#pragma unroll
            for (int u = 0; u < kUnroll; ++u)
                if (i0 + u * kStreamThreads < n) put_floats(s + at[u], v[u]);
        }
        __syncthreads();
        for (int i = tid; i < n; i += kStreamThreads) {
            const int j = i / nv, o = (i - j * nv) * V;
            const int r = r0 + j * (int)gridDim.x;
            const int orow = row_map ? row_map[r] : r;
            const float* sj = s + (size_t)j * bins * cs;
            int c = o / bins, b = o - c * bins;
            float w[V];
#pragma unroll
            for (int e = 0; e < V; ++e) {
                if (b == bins) { b = 0; ++c; }
                w[e] = sj[b * cs + c];
                ++b;
            }
            float* d = a.out + (size_t)orow * C * bins + o;
            if constexpr (V == 4) st_hint(d, make_float4(w[0], w[1], w[2], w[3]), norm);
            else st_hint(d, w[0], norm);
        }
        __syncthreads();
    }
}

template <int SR, int M>
__global__ void __launch_bounds__(kStreamThreads, 1)
roi_align_stream_fwd(const StreamArgs a) {
    constexpr int RB = 128 * (32 * M + 1);                        // bytes of one ring slot
    extern __shared__ unsigned char smem_raw[];
    // dynamic shared memory: the mbarriers -- full[k] at bars + 8k (32 arrivals: the lanes of the producer warp that staged the
    // row), empty[k] at bars + 8 * (kMaxSlots + k) (one arrival per consumer warp) -- then the ring (K logical slots + one
    // mirror of slot 0 behind slot K - 1, so that row y + 1 is always the next physical slot) and the per-warp table buffers,
    // whose space the tail reuses for the row blocks it transposes
    const unsigned bars = (smem_addr(smem_raw) + 127u) & ~127u;
    const unsigned ring = bars + kBarBytes;
    unsigned char* ring_ptr = smem_raw + (ring - smem_addr(smem_raw));
    const int tid = threadIdx.x;

    {   // the ring starts zeroed: a tap with weight 0 may read a slot that was never written (clamped last row)
        const int n16 = (a.K + 1) * (RB / 16);
        float4* r4 = reinterpret_cast<float4*>(ring_ptr);
        for (int k = tid; k < n16; k += kStreamThreads) r4[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (tid == 0) {
        for (int k = 0; k < a.K; ++k) { mbar_init(bars + 8u * k, 32u); mbar_init(bars + 8u * (kMaxSlots + k), kConsumerWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");             // the prepass's results are visible from here on
    // Everything the prepass wrote is read with ld.volatile / ld.cg from here on, never __ldg: a read-only (.nc) load carries
    // no dependence on the wait above and may be hoisted above it (DESIGN.md 4.1)
    int L0, L1;
    asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(L0) : "l"(a.piece_start + blockIdx.x) : "memory");
    asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(L1) : "l"(a.piece_start + blockIdx.x + 1) : "memory");
    stream_fragments<SR, M>(a, ring, bars, L0, L1);

    // ---- tail: once every CTA has stored its fragments (the grid is resident: see the launcher), transpose the rows
    asm volatile("cp.async.wait_all;" ::: "memory");
    prepass::grid_barrier(a.ticket);
    float* blocks = reinterpret_cast<float*>(ring_ptr);
    if ((a.C & 3) == 0 && (reinterpret_cast<uintptr_t>(a.out) & 15u) == 0) transpose_rows<4>(a, blocks);
    else transpose_rows<1>(a, blocks);
}

// ------------------------------------------------------------------------------------------------
// host: geometry, workspace, tensor map, launches
// ------------------------------------------------------------------------------------------------
size_t align_up_sz(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct StreamLayout {
    size_t ytab_off, xtab_off, zero_off, zero_bytes, rowptr_off, piece_off, entries_off, tmp_off, tmpcnt_off, ws_bytes;
    size_t prep_smem;           // dynamic shared memory of stream_prep
};

// One launch serves `levels` feature maps (FPN: the pyramid levels of one head; a plain call: one map).  All levels share the
// batch size, the channel count, the pooled size, the ring geometry (SX, K) and therefore the kernel instantiation.
// level_roi_begin: [levels + 1] first RoI of every level (RoIs are stored level-major), level_roi_begin[levels] = R.
bool stream_geometry(int levels, const float* const* bottoms, const int* heights, const int* widths, const float* scales,
                     const int* level_roi_begin, int N, int R, int C, int PH, int PW, int sr, int sm_count, StreamGeom* g,
                     StreamLayout* lay, unsigned* smem_bytes) {
    if (levels < 1 || levels > kMaxLevels) return false;
    if (sr < 1 || sr > 2 || PH * sr > kAxisMaxS || PW * sr > kAxisMaxS || PH > 31 || PW > 31) return false;
    if (N <= 0 || R <= 0 || R > 65535) return false;
    if ((long long)R * PH * PW * sr * sr >= (1LL << 28)) return false;
    for (int l = 0; l < levels; ++l)
        if (heights[l] < 2 || widths[l] < 2 || heights[l] > 65535) return false;
    // ring budget: everything but the per-warp table buffers, the barriers and the alignment slack
    const unsigned tabs = kConsumerWarps * kTabWords * 4;
    const unsigned ring_budget = kSmemBudget - tabs - kBarBytes - 128;
    int best_sx = 0, best_wx = 0, best_k = 0;
    long best_score = -1;
    for (int m = 1; m <= 3; ++m) {                            // SX = 32 m + 1: odd channel stride, m coalesced chunks + 1 column
        const int sx = 32 * m + 1;
        int k = (int)(ring_budget / (128u * (unsigned)sx)) - 1;       // one physical slot is the mirror of slot 0
        if (k > kMaxSlots) k = kMaxSlots;
        if (k < 12) continue;
        const int hx = m >= 2 ? 9 : 5;                        // halo: bins whose x samples are <= hx + 1 cells apart stay whole
        const int wx = sx - 1 - hx;
        long score = 0;                                       // columns staged per row of every level, weighted by its rows
        for (int l = 0; l < levels; ++l) {
            int s = 1;
            while ((s - 1) * wx + sx < widths[l]) ++s;        // the last strip needs no halo
            score += (long)s * sx * heights[l];
        }
        if (best_score < 0 || score < best_score) { best_score = score; best_sx = sx; best_wx = wx; best_k = k; }
    }
    if (best_score < 0) return false;
    // the main kernel's tail transposes whole output rows in shared memory: the ring's and the table buffers' space, or more
    // when one row block needs it
    const unsigned long long block = (unsigned long long)PH * PW * tail_stride(C) * 4u;
    if (block > kSmemBudget - kBarBytes - 128) return false;
    const unsigned ring_bytes = (unsigned)(best_k + 1) * 128u * (unsigned)best_sx + tabs;
    const unsigned tail_bytes = ring_bytes > block ? ring_bytes : (unsigned)block;
    g->tail_rows = (int)(tail_bytes / block);
    g->N = N; g->R = R; g->C = C; g->PH = PH; g->PW = PW; g->sr = sr;
    g->ny = PH * sr; g->nx = PW * sr;
    g->SX = best_sx; g->WX = best_wx; g->K = best_k;
    g->row_bytes = 128 * best_sx;
    g->L = levels;
    int q = 0;
    long long keys = 0;
    for (int l = 0; l < levels; ++l) {
        StreamLevel& lv = g->lv[l];
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
        if (keys >= (1LL << 24)) return false;
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
    // the prepass scans the keys in shared memory
    lay->prep_smem = (size_t)2 * (g->keys + 1) * 4 + (size_t)g->cap_r * 12;
    if (lay->prep_smem > kPrepSmemMax) return false;
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
    *smem_bytes = kBarBytes + tail_bytes + 128;
    return true;
}

size_t stream_fpn_workspace_bytes(int levels, const int* heights, const int* widths, int N, int R, int PH, int PW, int sr) {
    StreamGeom g;
    StreamLayout lay;
    unsigned smem = 0;
    if (!stream_geometry(levels, nullptr, heights, widths, nullptr, nullptr, N, R, 32, PH, PW, sr, kNumSMs, &g, &lay, &smem)) return 0;
    return lay.ws_bytes;
}

// One launch sequence over the level table (a plain call is one level).  Returns B200_ROI_OK when the streaming path ran;
// kPathDeclined when it does not apply (caller falls back).
int roi_align_forward_stream_fpn(int levels, const float* const* bottoms, const int* heights, const int* widths, const float* scales,
                                 const int* level_roi_begin, int N, int R, int C, int PH, int PW, int sr, const float* rois, float* top,
                                 const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    if (workspace == nullptr || C <= 0) return kPathDeclined;
    if ((long long)N * C >= (1LL << 31) || (long long)R * C * PH * PW >= (1LL << 31)) return kPathDeclined;
    int sm_count = 0;
    if (device_sm_count(&sm_count) != B200_ROI_OK) return kPathDeclined;
    StreamGeom g;
    StreamLayout lay;
    unsigned smem = 0;
    if (!stream_geometry(levels, bottoms, heights, widths, scales, level_roi_begin, N, R, C, PH, PW, sr, sm_count, &g, &lay, &smem)) return kPathDeclined;
    if (workspace_bytes < lay.ws_bytes) return kPathDeclined;
    unsigned char* wsb = (unsigned char*)workspace;
    StreamWs ws;
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

    const int m = (g.SX - 1) / 32;
    const auto prep = sr == 1 ? stream_prep<1> : stream_prep<2>;
    const auto fwd = sr == 1 ? (m == 1 ? roi_align_stream_fwd<1, 1> : m == 2 ? roi_align_stream_fwd<1, 2> : roi_align_stream_fwd<1, 3>)
                             : (m == 1 ? roi_align_stream_fwd<2, 1> : m == 2 ? roi_align_stream_fwd<2, 2> : roi_align_stream_fwd<2, 3>);
    if (smem_opt_in(prep, kPrepSmemMax) != B200_ROI_OK || smem_opt_in(fwd, kSmemBudget) != B200_ROI_OK) return kPathDeclined;
    // prepass grid: one CTA per RoI when they are all resident at once (the kernel has a grid barrier), else a resident grid
    int per_sm = 0;
    cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, prep, kPrepThreads, lay.prep_smem);
    if (err != cudaSuccess || per_sm < 1) { (void)cudaGetLastError(); return kPathDeclined; }
    const long long cap = (long long)per_sm * sm_count;
    const int prep_grid = (int)(R < cap ? R : cap);
    const int n16 = (int)(lay.zero_bytes / 16);
    // the main kernel has a grid barrier too: one CTA per SM must be resident at its shared-memory size
    err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fwd, kStreamThreads, smem);
    if (err != cudaSuccess || (long long)per_sm * sm_count < g.pieces) { (void)cudaGetLastError(); return kPathDeclined; }

    StreamArgs a;
    a.ytab = ws.ytab; a.xtab = ws.xtab; a.entries = ws.entries; a.rowptr = ws.rowptr; a.maxend = ws.maxend;
    a.piece_start = ws.piece_start; a.out = top; a.row_map = row_map; a.ticket = ws.ticket + 1;
    a.R = R; a.tail_rows = g.tail_rows;
    a.C = C; a.G = g.G; a.K = g.K; a.WX = g.WX; a.PH = PH; a.PW = PW; a.ny = g.ny; a.nx = g.nx; a.L = g.L; a.Q = g.Q;
    for (int l = 0; l < kMaxLevels; ++l) a.lv[l] = g.lv[l];
    for (int c = 0; c <= kMaxCols; ++c) a.colstart[c] = g.colstart[c];

    // clear -> prep -> main, each launched as the programmatic dependent of the one before (it starts once every CTA of the
    // previous kernel has signalled launch_dependents, and waits for that kernel's results with griddepcontrol.wait)
    stream_clear<<<(n16 + kPrepThreads - 1) / kPrepThreads, kPrepThreads, 0, stream>>>((int4*)zero, n16);
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)prep_grid);
    cfg.blockDim = dim3(kPrepThreads);
    cfg.dynamicSmemBytes = lay.prep_smem;
    cfg.stream = stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    err = cudaLaunchKernelEx(&cfg, prep, rois, g, ws, top, row_map);
    if (err != cudaSuccess) return (int)err;
    cfg.gridDim = dim3((unsigned)g.pieces);
    cfg.blockDim = dim3(kStreamThreads);
    cfg.dynamicSmemBytes = smem;
    err = cudaLaunchKernelEx(&cfg, fwd, a);
    if (err != cudaSuccess) return (int)err;
    return finish_launch(3);
}

}  // namespace

void roi_align_stream_set_debug_buffer(unsigned long long* host_pinned) {
    cudaMemcpyToSymbol(g_stream_dead, &host_pinned, sizeof(host_pinned));      // [CTA][32] u64 watchdog records
}

size_t roi_align_stream_workspace_bytes(int N, int R, int H, int W, int PH, int PW, int sr) {
    return stream_fpn_workspace_bytes(1, &H, &W, N, R, PH, PW, sr);
}

// returns B200_ROI_OK when the streaming path ran; kPathDeclined when it does not apply (caller falls back)
int roi_align_forward_stream(const float* bottom, float scale, int N, int R, int H, int W, int C, int PH, int PW, int sr,
                             const float* rois, float* top, const int* row_map, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    const int begin[2] = {0, R};
    return roi_align_forward_stream_fpn(1, &bottom, &H, &W, &scale, begin, N, R, C, PH, PW, sr, rois, top, row_map, workspace,
                                        workspace_bytes, stream);
}

}  // namespace b200
