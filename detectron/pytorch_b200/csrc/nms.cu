// nms.cu -- proposal-layer NMS, everything on the device and on the caller's stream.
//
// Semantics: lib/model/nms/src/nms_cuda_kernel.cu (reference) devIoU :31-39, nms_kernel :41-85,
// host greedy scan :123-144.  Kept indices are bit-exact with the reference because (a) the IoU
// test reproduces the reference's SASS rounding recipe (row box = lower index: rounded area Sa;
// column box area fused: FFMA(bw, bh, Sa); IEEE division; strict '>') and (b) the greedy scan is
// the same integer logic -- box j is dropped iff a kept box i < j has bit (i, j) set.
//
// Differences in mechanism (not in results): only the upper triangle of 64x64 tiles is computed
// (the reference commented its triangular skip out, :46, and did 2x the work), with a division-free
// fast path for the IoU test and the exact recipe for the pairs it cannot settle; the suppression
// scan runs on the GPU (one CTA: a resolver warp walks the 64-box diagonal blocks, 24 worker warps
// fold the kept rows into the running removal words behind it) instead of a 4.5 MB blocking D2H
// copy + single-threaded CPU loop + H2D; no cudaMalloc/cudaFree: scratch comes from the caller.
#include "common.cuh"
#include <math.h>
#include <stdlib.h>

namespace b200 {

constexpr int kNmsTile = 64;
constexpr int kScanThreads = 1024;
constexpr int kFoldGroups = 2, kFoldWarps = 12;     // resolver scan: 2 blocks folded concurrently by 12 warps each (24 worker warps)

typedef unsigned long long u64;

// mbarrier handshakes (shared::cta): waiting warps are suspended by the hardware instead of polling shared memory
// (24 polling warps saturate the LSU queue the resolver's own shared loads go through).  arrive = release,
// try_wait = acquire at CTA scope, so no separate fences are needed around the flag.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(u64* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(u64* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "MBAR_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra MBAR_DONE;\n"
        "bra MBAR_WAIT;\n"
        "MBAR_DONE:\n"
        "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

struct __align__(16) ColBox {
    float x0, y0, x1, y1;
};

// The exact IoU test of one pair (a = the higher-scoring "row" box, Sa its rounded area).  Two flavours:
//   CUDA   (kCython = false): the reference CUDA kernel's recipe, den = FFMA(bw, bh, Sa) - inter, suppress on IoU > thresh;
//   Cython (kCython = true):  lib/utils/cython_nms.pyx:37-87, both areas rounded on their own, den = (Sa + Sb) - inter,
//                             suppress on IoU >= thresh.
template <bool kCython>
__device__ __forceinline__ bool nms_bit(float a0, float a1, float a2, float a3, float Sa,
                                        float b0, float b1, float b2, float b3, float thresh) {
    const float left = fmaxf(a0, b0), right = fminf(a2, b2);
    const float top = fmaxf(a1, b1), bottom = fminf(a3, b3);
    const float w = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.f), 0.f);
    const float h = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.f), 0.f);
    const float inter = __fmul_rn(w, h);
    const float bw = __fadd_rn(__fsub_rn(b2, b0), 1.f), bh = __fadd_rn(__fsub_rn(b3, b1), 1.f);
    if (kCython) return __fdiv_rn(inter, __fsub_rn(__fadd_rn(Sa, __fmul_rn(bw, bh)), inter)) >= thresh;
    return __fdiv_rn(inter, __fsub_rn(__fmaf_rn(bw, bh, Sa), inter)) > thresh;
}

struct __align__(16) ColBoxEx {
    float x0, y0, x1, y1;
    float bw, bh, pad0, pad1;           // (x1 - x0) + 1, (y1 - y0) + 1: the operands of the fused column-box area
};

// One CTA per 64x64 tile of the upper triangle (linear tile index: the diagonal tiles, which also produce the
// transposed words, come first).  The IoU test is decided without the IEEE division whenever that is safe:
// q' = inter * rcp.approx(den) is within 2^-21 (relative) of the correctly rounded quotient once den is a positive
// normal number well inside the exponent range, so q' > thresh (1 + 2^-18) or q' < thresh (1 - 2^-18) settles the
// comparison; everything else (the band around the threshold, den <= 0 / tiny / huge / NaN, thresholds outside
// [2^-20, 2^20]: lo = -inf, hi = +inf) is marked undecided and re-evaluated with the exact recipe (nms_bit) after
// the main loop.  Results are therefore bit-identical to the all-division version; the main loop is branch-free,
// fully unrolled (bit positions are immediates) and ~26 instructions per pair instead of ~42.
// The screen serves both flavours of nms_bit: their denominators differ by about one rounding, far inside the band, and
// `>` and `>=` differ only at the threshold itself, so only the exact re-evaluation and the transposed words depend on it.
template <bool kCython>
__device__ __forceinline__ void nms_mask_tile(const float* __restrict__ boxes, int n, int dim, float thresh, float lo, float hi,
                                              u64* __restrict__ mask, u64* __restrict__ diag_t, int idx) {
    const int col_blocks = (n + kNmsTile - 1) / kNmsTile;
    int row_start, col_start;
    {
        if (idx < col_blocks) {
            row_start = col_start = idx;
        } else {                                    // k enumerates the pairs row < col: k = col (col - 1) / 2 + row
            const int k = idx - col_blocks;
            int c = (int)((1.f + sqrtf(1.f + 8.f * (float)k)) * 0.5f);
            while ((long long)c * (c - 1) / 2 > k) --c;
            while ((long long)(c + 1) * c / 2 <= k) ++c;
            col_start = c;
            row_start = k - (int)((long long)c * (c - 1) / 2);
        }
    }
    const int row_size = min(n - row_start * kNmsTile, kNmsTile);
    const int col_size = min(n - col_start * kNmsTile, kNmsTile);
    __shared__ ColBoxEx cols[kNmsTile];
    {
        ColBoxEx b; b.x0 = b.y0 = b.x1 = b.y1 = 0.f; b.pad0 = b.pad1 = 0.f;
        if ((int)threadIdx.x < col_size) {
            const float* p = boxes + (size_t)(col_start * kNmsTile + threadIdx.x) * dim;
            b.x0 = p[0]; b.y0 = p[1]; b.x1 = p[2]; b.y1 = p[3];
        }
        b.bw = __fadd_rn(__fsub_rn(b.x1, b.x0), 1.f);
        b.bh = __fadd_rn(__fsub_rn(b.y1, b.y0), 1.f);
        cols[threadIdx.x] = b;
    }
    __syncthreads();
    if ((int)threadIdx.x >= row_size) return;
    const int cur = row_start * kNmsTile + threadIdx.x;
    const float* a = boxes + (size_t)cur * dim;
    const float a0 = a[0], a1 = a[1], a2 = a[2], a3 = a[3];
    const float Sa = __fmul_rn(__fadd_rn(__fsub_rn(a2, a0), 1.f), __fadd_rn(__fsub_rn(a3, a1), 1.f));
    unsigned t_lo = 0u, t_hi = 0u, u_lo = 0u, u_hi = 0u;        // decided-true bits / undecided bits
    const float qnan = __int_as_float(0x7fc00000);
#pragma unroll
    for (int i = 0; i < kNmsTile; ++i) {
        const float4 bx = *reinterpret_cast<const float4*>(&cols[i].x0);
        const float2 bs = *reinterpret_cast<const float2*>(&cols[i].bw);
        const float left = fmaxf(a0, bx.x), right = fminf(a2, bx.z);
        const float top = fmaxf(a1, bx.y), bottom = fminf(a3, bx.w);
        const float w = fmaxf(__fadd_rn(__fsub_rn(right, left), 1.f), 0.f);
        const float h = fmaxf(__fadd_rn(__fsub_rn(bottom, top), 1.f), 0.f);
        const float inter = __fmul_rn(w, h);
        const float den = __fsub_rn(__fmaf_rn(bs.x, bs.y, Sa), inter);
        float r;
        asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(den));
        const bool in_range = (__float_as_uint(den) - 0x20800000u) < (0x5E800000u - 0x20800000u);     // 2^-62 <= den < 2^62
        const float q = in_range ? __fmul_rn(inter, r) : qnan;
        const bool yes = q > hi, decided = yes || (q < lo);
        if (i < 32) { if (yes) t_lo |= 1u << i; if (!decided) u_lo |= 1u << i; }
        else        { if (yes) t_hi |= 1u << (i - 32); if (!decided) u_hi |= 1u << (i - 32); }
    }
    u64 t = ((u64)t_hi << 32) | t_lo, und = ((u64)u_hi << 32) | u_lo;
    u64 live = (col_size == kNmsTile) ? ~0ULL : ((1ULL << col_size) - 1ULL);
    if (row_start == col_start) live &= ~((2ULL << threadIdx.x) - 1ULL);       // only columns above the own index
    t &= live; und &= live;
    while (und) {                                   // rare: exact evaluation of the pairs the fast test could not settle
        const int i = __ffsll((long long)und) - 1;
        und &= und - 1ULL;
        const ColBoxEx b = cols[i];
        if (nms_bit<kCython>(a0, a1, a2, a3, Sa, b.x0, b.y0, b.x1, b.y1, thresh)) t |= 1ULL << i;
    }
    mask[(size_t)cur * col_blocks + col_start] = t;
    if (row_start == col_start) {
        // Transposed diagonal word: bit j (< own index) <=> box j's mask word has this box's bit set.  Same function,
        // same operand roles (box j is the "row" box with the rounded area) as the thread of row j evaluates, so the
        // two are the same bits by construction.  Used by the resolver scan's parallel block resolve.
        u64 tt = 0;
        for (int j = 0; j < (int)threadIdx.x; ++j) {
            const ColBoxEx r = cols[j];
            if (nms_bit<kCython>(r.x0, r.y0, r.x1, r.y1, __fmul_rn(r.bw, r.bh), a0, a1, a2, a3, thresh)) tt |= 1ULL << j;
        }
        diag_t[cur] = tt;
    }
}

// ---- independent problems in one launch (SURVEY 8f N1: the (image, level) proposal sets of one step; b200_nms is one problem) ----
constexpr int kNmsMaxProblems = 64;
struct NmsBatch {
    int count;
    int n[kNmsMaxProblems];                     // boxes of problem p
    int box_off[kNmsMaxProblems];               // its first row in `boxes` / first slot in `keep_out`
    int tile_off[kNmsMaxProblems + 1];          // its first CTA of the mask launch
    unsigned long long mask_off[kNmsMaxProblems];       // word offsets into the workspace
    unsigned long long diag_off[kNmsMaxProblems];
};

template <bool kCython>
__global__ void __launch_bounds__(kNmsTile)
nms_mask_batched_kernel(const float* __restrict__ boxes, const __grid_constant__ NmsBatch nb, int dim, float thresh, float lo, float hi,
                        u64* __restrict__ ws) {
    int p = 0;                                  // problem of this CTA: tile_off is ascending
    {
        int lo_p = 0, hi_p = nb.count - 1;
        while (lo_p < hi_p) {
            const int mid = (lo_p + hi_p + 1) >> 1;
            if (nb.tile_off[mid] <= (int)blockIdx.x) lo_p = mid; else hi_p = mid - 1;
        }
        p = lo_p;
    }
    nms_mask_tile<kCython>(boxes + (size_t)nb.box_off[p] * dim, nb.n[p], dim, thresh, lo, hi, ws + nb.mask_off[p], ws + nb.diag_off[p],
                  (int)blockIdx.x - nb.tile_off[p]);
}

// Single-CTA greedy scan over the upper-triangular mask.  remv[] (one 64-bit word per column block)
// lives in shared memory.
__global__ void __launch_bounds__(kScanThreads)
nms_scan_kernel(const u64* __restrict__ mask, int n, int col_blocks, int* __restrict__ keep_out, int* __restrict__ num_out) {
    extern __shared__ u64 remv[];
    __shared__ u64 s_kept;
    __shared__ int s_count;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int j = tid; j < col_blocks; j += kScanThreads) remv[j] = 0;
    if (tid == 0) s_count = 0;
    __syncthreads();

    for (int b = 0; b < col_blocks; ++b) {
        const int lim = min(kNmsTile, n - b * kNmsTile);
        if (warp == 0) {
            // lane l holds the diagonal words of rows b*64 + l and b*64 + 32 + l
            const int r0 = b * kNmsTile + lane, r1 = r0 + 32;
            const u64 d_lo = (r0 < n) ? mask[(size_t)r0 * col_blocks + b] : 0;
            const u64 d_hi = (r1 < n) ? mask[(size_t)r1 * col_blocks + b] : 0;
            u64 r = remv[b];
            u64 kept = 0;
#pragma unroll 8
            for (int k = 0; k < kNmsTile; ++k) {
                const u64 dk = __shfl_sync(0xffffffffu, (k < 32) ? d_lo : d_hi, k & 31);
                if (k < lim && !((r >> k) & 1ULL)) { kept |= 1ULL << k; r |= dk; }
            }
            if (lane == 0) s_kept = kept;
        }
        __syncthreads();
        const u64 kept = s_kept;
        const int base = s_count;
        if (tid < kNmsTile && ((kept >> tid) & 1ULL))
            keep_out[base + __popcll(kept & ((1ULL << tid) - 1ULL))] = b * kNmsTile + tid;
        // OR the mask rows of the kept boxes of block b into remv[j], j > b:
        // thread = (k-group of 8, column word j); 128 column words per pass.
        const int kg = tid >> 7;            // 0..7
        for (int j = b + 1 + (tid & 127); j < col_blocks; j += 128) {
            u64 acc = 0;
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const int k = kg + 8 * kk;
                if ((kept >> k) & 1ULL) acc |= mask[(size_t)(b * kNmsTile + k) * col_blocks + j];
            }
            if (acc) atomicOr(&remv[j], acc);
        }
        __syncthreads();
        if (tid == 0) s_count = base + __popcll(kept);
        // (next iteration's first __syncthreads publishes s_count / remv)
    }
    __syncthreads();
    if (tid == 0) *num_out = s_count;
}

// Resolver scan (default while REACH * n * 8 B fits shared memory).  Everything the greedy chain itself touches is
// copied to shared memory once, so the single resolver warp never waits for global memory:
//   * T[i]   -- the TRANSPOSED diagonal word of box i (which earlier boxes of its own 64-block suppress it), and
//   * D[t][i] -- the mask words t = 1 .. REACH-1 column blocks right of the diagonal.
// A block is resolved in parallel, lanes = boxes (two per lane), by iterating to the fixed point of the greedy rule:
// an undecided box whose in-block suppressors are all removed is kept; one with a kept suppressor is removed.  The
// lowest undecided box is decided in every round, so this terminates with exactly the sequential result; the number
// of rounds is the longest suppression chain inside the block (2-4 for proposal-like inputs, 64 at worst) instead of
// 64 dependent steps.  The resolver then derives from its own kept rows the contribution to the next REACH-1 column
// blocks.  24 worker warps (2 groups x 12) fold the kept rows into the remaining columns (j >= block + REACH) from
// global memory, lanes = columns (coalesced 256-byte row segments, 8 rows in flight per warp); the resolver
// only checks that the block REACH steps back has been folded.
template <int REACH>
__device__ __forceinline__ void nms_scan_resolver_body(const u64* __restrict__ mask, const u64* __restrict__ diag_t, int n, int col_blocks,
                                                       int* __restrict__ keep_out, int* __restrict__ num_out) {
    extern __shared__ u64 sm[];
    const int n_pad = col_blocks * kNmsTile;
    u64* D = sm;                                    // D[0][i] = T[i]; D[t][i] = mask[i][blk(i) + t], 1 <= t < REACH
    u64* remv = D + (size_t)REACH * n_pad;          // [col_blocks]  contributions of blocks <= j - REACH (workers, smem atomics)
    u64* kept_hist = remv + col_blocks;             // [col_blocks]
    u64* res_bar = kept_hist + col_blocks;          // [col_blocks] mbarrier: block resolved (1 arrival, resolver lane 0)
    u64* fold_bar = res_bar + col_blocks;           // [col_blocks] mbarrier: block folded (kFoldWarps arrivals)
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    for (int i = tid; i < n_pad; i += kScanThreads) {
        const int cbk = i >> 6;
        const u64* row = mask + (size_t)i * col_blocks + cbk;
        D[i] = (i < n) ? diag_t[i] : 0ULL;
#pragma unroll
        for (int t = 1; t < REACH; ++t) D[(size_t)t * n_pad + i] = (i < n && cbk + t < col_blocks) ? row[t] : 0ULL;
    }
    for (int j = tid; j < col_blocks; j += kScanThreads) { remv[j] = 0; mbar_init(&res_bar[j], 1); mbar_init(&fold_bar[j], kFoldWarps); }
    __syncthreads();

    if (warp == 0) {
        u64 c[REACH];                               // c[t]: contribution of already resolved blocks to column b + t (t >= 1)
#pragma unroll
        for (int t = 0; t < REACH; ++t) c[t] = 0;
        int count = 0;
        const u64 bit0 = 1ULL << lane, bit1 = 1ULL << (lane + 32);
        for (int b = 0; b < col_blocks; ++b) {
            const u64 T0 = D[b * kNmsTile + lane], T1 = D[b * kNmsTile + lane + 32];
            if (b >= REACH) mbar_wait(&fold_bar[b - REACH], 0);
            const int lim = min(kNmsTile, n - b * kNmsTile);
            u64 rem = *reinterpret_cast<volatile u64*>(&remv[b]) | c[1];
            if (lim < kNmsTile) rem |= ~((1ULL << lim) - 1ULL);       // padded rows: decided, never kept
            u64 kept = 0;
            while ((kept | rem) != ~0ULL) {
                const u64 dec = kept | rem;
                const bool u0 = !(dec & bit0), u1 = !(dec & bit1);
                const bool nk0 = u0 && !(T0 & ~rem), nk1 = u1 && !(T1 & ~rem);      // every suppressor already removed
                const bool nr0 = u0 && (T0 & kept), nr1 = u1 && (T1 & kept);        // suppressed by a kept box
                const unsigned k_lo = __ballot_sync(0xffffffffu, nk0), k_hi = __ballot_sync(0xffffffffu, nk1);
                const unsigned r_lo = __ballot_sync(0xffffffffu, nr0), r_hi = __ballot_sync(0xffffffffu, nr1);
                kept |= ((u64)k_hi << 32) | k_lo;
                rem |= ((u64)r_hi << 32) | r_lo;
            }
            if (lane == 0) { kept_hist[b] = kept; mbar_arrive(&res_bar[b]); }
            // contributions of this block's kept rows to the next REACH-1 columns; shift the carries by one column
            const bool ka = (kept >> lane) & 1ULL, kb2 = (kept >> (lane + 32)) & 1ULL;
#pragma unroll
            for (int t = 1; t < REACH; ++t) {
                u64 v = 0;
                if (ka) v = D[(size_t)t * n_pad + b * kNmsTile + lane];
                if (kb2) v |= D[(size_t)t * n_pad + b * kNmsTile + lane + 32];
                const unsigned lo = __reduce_or_sync(0xffffffffu, (unsigned)v);
                const unsigned hi = __reduce_or_sync(0xffffffffu, (unsigned)(v >> 32));
                const u64 kt = ((u64)hi << 32) | lo;
                c[t] = ((t + 1 < REACH) ? c[t + 1] : 0ULL) | kt;
            }
            const u64 lo_mask = (1ULL << lane) - 1ULL;
            if (ka) keep_out[count + __popcll(kept & lo_mask)] = b * kNmsTile + lane;
            if (kb2) keep_out[count + __popcll(kept & ((lo_mask << 32) | 0xffffffffULL))] = b * kNmsTile + lane + 32;
            count += __popcll(kept);
        }
        if (lane == 0) *num_out = count;
    } else if ((warp & 3) != 0) {
        // Workers sit on warp slots with (warp & 3) != 0: warp w issues from scheduler w & 3, so the resolver warp has
        // scheduler 0 to itself and its dependent chain is never delayed by the workers' polling loops.  Group g folds
        // blocks b = g, g+2, ...; the block's (32-column chunk, 16-row part) units are dealt round-robin to its 12 warps.
        // Shared-memory merges are 32-bit atomics (a 64-bit shared atomicOr is a CAS loop).
        const int ww = (warp >> 2) * 3 + (warp & 3) - 1;
        const int g = ww / kFoldWarps, wi = ww - g * kFoldWarps;
        unsigned* remv32 = reinterpret_cast<unsigned*>(remv);
        for (int b = g; b < col_blocks; b += kFoldGroups) {
            mbar_wait(&res_bar[b], 0);
            const u64 kept = *reinterpret_cast<volatile u64*>(&kept_hist[b]);
            const int ncols = col_blocks - (b + REACH);
            if (ncols > 0) {
                const int nchunks = (ncols + 31) >> 5;
                constexpr int part_shift = 2;                             // 4 row parts of 16 rows: <= 12 units for <= 96 columns
                const int rows_per = kNmsTile >> part_shift;
                const int units = nchunks << part_shift;
                for (int u = wi; u < units; u += kFoldWarps) {
                    const int cch = u >> part_shift, part = u & ((1 << part_shift) - 1);
                    unsigned kb = (unsigned)(kept >> (part * rows_per));
                    if (rows_per < 32) kb &= (1u << rows_per) - 1u;
                    const int j = b + REACH + cch * 32 + lane;
                    const bool jok = j < col_blocks;
                    const u64* base = mask + (size_t)(b * kNmsTile + part * rows_per) * col_blocks + (jok ? j : 0);
                    u64 acc = 0;
                    if (jok) {
                        // all 16 rows of the part in flight at once; the address walks down the rows so that it
                        // lives in one register pair instead of sixteen
                        u64 v[16];
                        const u64* p = base;
#pragma unroll
                        for (int t = 0; t < 16; ++t) {
                            v[t] = ((kb >> t) & 1u) ? *p : 0ULL;
                            p += col_blocks;
                        }
#pragma unroll
                        for (int t = 0; t < 16; ++t) acc |= v[t];
                    }
                    if (jok) {
                        const unsigned lo = (unsigned)acc, hi = (unsigned)(acc >> 32);
                        if (lo) atomicOr(&remv32[2 * j], lo);
                        if (hi) atomicOr(&remv32[2 * j + 1], hi);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&fold_bar[b]);
        }
    }
}

// one CTA per problem
template <int REACH>
__global__ void __launch_bounds__(kScanThreads)
nms_scan_resolver_batched_kernel(const u64* __restrict__ ws, const __grid_constant__ NmsBatch nb, int* __restrict__ keep_out,
                                 int* __restrict__ num_out) {
    const int p = blockIdx.x;
    const int n = nb.n[p];
    if (n == 0) { if (threadIdx.x == 0) num_out[p] = 0; return; }
    nms_scan_resolver_body<REACH>(ws + nb.mask_off[p], ws + nb.diag_off[p], n, (n + kNmsTile - 1) / kNmsTile, keep_out + nb.box_off[p],
                                  num_out + p);
}

__global__ void nms_empty_kernel(int* num_out) { *num_out = 0; }

// ---- batched entry: `num_problems` independent score-sorted box sets, stored back to back in `boxes` ----
static bool nms_batch_plan(const int* counts, int num_problems, NmsBatch* nb, size_t* ws_words, int* max_n) {
    if (num_problems < 1 || num_problems > kNmsMaxProblems) return false;
    nb->count = num_problems;
    long long box = 0, tile = 0;
    size_t words = 0;
    int mx = 0;
    for (int p = 0; p < num_problems; ++p) {
        const int n = counts[p];
        if (n < 0) return false;
        const long long cb = (n + kNmsTile - 1) / kNmsTile;
        nb->n[p] = n; nb->box_off[p] = (int)box; nb->tile_off[p] = (int)tile;
        nb->mask_off[p] = words; words += (size_t)n * cb;
        nb->diag_off[p] = words; words += (size_t)cb * kNmsTile;
        box += n; tile += cb * (cb + 1) / 2;
        if (box > 0x7fffffffLL || tile > 0x7fffffffLL) return false;
        if (n > mx) mx = n;
    }
    nb->tile_off[num_problems] = (int)tile;
    for (int p = num_problems; p < kNmsMaxProblems; ++p) { nb->n[p] = 0; nb->box_off[p] = (int)box; nb->tile_off[p + 1] = (int)tile; nb->mask_off[p] = nb->diag_off[p] = words; }
    *ws_words = words; *max_n = mx;
    return true;
}

// cython: the IoU test of lib/utils/cython_nms.pyx (see nms_bit) instead of the reference CUDA kernel's
static int nms_batched(const float* boxes, const int* counts, int num_problems, int dim, float thresh, bool cython, int* keep_out,
                       int* num_out, void* workspace, size_t workspace_bytes, cudaStream_t stream) {
    if (!counts || num_problems < 1 || !num_out) return B200_ROI_EINVAL;
    long long total = 0;
    for (int p = 0; p < num_problems && p < 64; ++p) total += counts[p] > 0 ? counts[p] : 0;
    if (total > 0 && (!boxes || !keep_out)) return B200_ROI_EINVAL;
    NmsBatch nb; size_t words = 0; int mx = 0;
    if (dim < 4 || !nms_batch_plan(counts, num_problems, &nb, &words, &mx)) return B200_ROI_EINVAL;
    if (workspace == nullptr || workspace_bytes < (words * sizeof(u64) + 255) / 256 * 256) return B200_ROI_EWORKSPACE;
    float lo = -INFINITY, hi = INFINITY;
    if (thresh >= 9.5367431640625e-07f && thresh <= 1048576.f) {
        lo = (float)((double)thresh * (1.0 - 3.814697265625e-06));
        hi = (float)((double)thresh * (1.0 + 3.814697265625e-06));
    }
    const int cb = (mx + kNmsTile - 1) / kNmsTile;
    int reach = 0;
    size_t smem_res = 0;
    for (int r = 4; r >= 2; --r) {
        const size_t sm_r = sizeof(u64) * ((size_t)r * cb * kNmsTile + 4 * (size_t)cb) + 16;
        if (sm_r <= 224 * 1024) { reach = r; smem_res = sm_r; break; }
    }
    u64* ws = (u64*)workspace;
    if (nb.tile_off[num_problems] > 0)
        (cython ? nms_mask_batched_kernel<true> : nms_mask_batched_kernel<false>)<<<(unsigned)nb.tile_off[num_problems], kNmsTile, 0, stream>>>(
            boxes, nb, dim, thresh, lo, hi, ws);
    if (reach == 0) {
        // a problem too large for the pipelined scan (> ~13.8k boxes): the unpipelined scan, one launch per problem
        if (const int rc = smem_opt_in(nms_scan_kernel, sizeof(u64) * (size_t)cb)) return rc;
        for (int p = 0; p < num_problems; ++p) {
            const int n = nb.n[p];
            if (n == 0) nms_empty_kernel<<<1, 1, 0, stream>>>(num_out + p);
            else nms_scan_kernel<<<1, kScanThreads, sizeof(u64) * (size_t)((n + kNmsTile - 1) / kNmsTile), stream>>>(
                ws + nb.mask_off[p], n, (n + kNmsTile - 1) / kNmsTile, keep_out + nb.box_off[p], num_out + p);
        }
        return finish_launch(1 + num_problems);
    }
    void (*kern)(const u64*, const NmsBatch, int*, int*) =
        (reach == 4) ? nms_scan_resolver_batched_kernel<4> : (reach == 3) ? nms_scan_resolver_batched_kernel<3> : nms_scan_resolver_batched_kernel<2>;
    if (const int rc = smem_opt_in(kern, smem_res)) return rc;
    kern<<<num_problems, kScanThreads, smem_res, stream>>>(ws, nb, keep_out, num_out);
    return finish_launch(2);
}

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_nms_workspace_bytes(int n) {
    if (n <= 0) return 256;
    const size_t cb = (size_t)(n + kNmsTile - 1) / kNmsTile;
    return (((size_t)n * cb + cb * kNmsTile) * sizeof(u64) + 255) / 256 * 256;     // mask words + transposed diagonal words
}

int b200_nms(const float* boxes, int n, int dim, float thresh, int* keep_out, int* num_out, void* workspace,
             size_t workspace_bytes, b200_stream_t stream) {
    if (!num_out || (n > 0 && (!boxes || !keep_out))) return B200_ROI_EINVAL;
    if (n < 0 || dim < 4) return B200_ROI_EINVAL;
    if (n == 0) {
        nms_empty_kernel<<<1, 1, 0, stream>>>(num_out);
        return finish_launch();
    }
    if (workspace == nullptr || workspace_bytes < b200_nms_workspace_bytes(n)) return B200_ROI_EWORKSPACE;
    // a batch of one problem: its mask words start at the workspace and its transposed diagonal words follow them, the
    // layout b200_nms_workspace_bytes sizes
    return nms_batched(boxes, &n, 1, dim, thresh, false, keep_out, num_out, workspace, workspace_bytes, stream);
}

size_t b200_nms_batched_workspace_bytes(const int* counts, int num_problems) {
    if (!counts) return 0;
    NmsBatch nb; size_t words = 0; int mx = 0;
    if (!nms_batch_plan(counts, num_problems, &nb, &words, &mx)) return 0;
    return (words * sizeof(u64) + 255) / 256 * 256 + 256;
}

int b200_nms_batched(const float* boxes, const int* counts, int num_problems, int dim, float thresh, int* keep_out, int* num_out,
                     void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    return nms_batched(boxes, counts, num_problems, dim, thresh, false, keep_out, num_out, workspace, workspace_bytes, stream);
}

int b200_nms_batched_cython(const float* boxes, const int* counts, int num_problems, int dim, float thresh, int* keep_out, int* num_out,
                            void* workspace, size_t workspace_bytes, b200_stream_t stream) {
    return nms_batched(boxes, counts, num_problems, dim, thresh, true, keep_out, num_out, workspace, workspace_bytes, stream);
}

}  // extern "C"
