// jpeg.cu -- baseline JPEG decode (cv2.imread / cv2.imdecode with IMREAD_COLOR, bit for bit) for all images of a call in
// three launches.  The host (utils/jpeg.py) has parsed the headers, derived the Huffman decode tables and cut each scan into
// its restart intervals with the byte stuffing removed; oracle/jpeg.py restates every step in numpy.
//
// 1. jpeg_huffman_kernel, one CTA per restart interval: parallel Huffman decode by self-synchronisation.  The interval's L bits
//    are cut into subsequences of S bits; thread t owns the contiguous run of subsequences [t R, (t + 1) R), R = ceil(n / T).
//    A decoder state at a codeword boundary is (bit offset, block within the MCU, coefficient index k).
//    a. Every thread decodes its run; its first subsequence starts from a guess (its first bit, block 0, k = 0), the others
//       from the exit state of the one before.  in[j] / out[j] record each subsequence's entry and exit state and block count.
//       JPEG's Huffman codes resynchronise quickly (Klein & Wiseman 2003), so a guessed decode soon meets the true one.
//    b. Sync passes: thread t compares the exit state of run t - 1 with its own entry state; on a difference it decodes again
//       from that state and stops at the first subsequence whose new entry state equals the recorded one.  Each pass makes at
//       least one more run exact: a run that never syncs is decoded as the sequential decoder would, slower, never wrong.
//    c. A block scan of the runs' block counts gives each run its first block; a last exit state other than (L, 0, 0), an error
//       in a subsequence's exact decode (a bad code, a code past the interval, a coefficient index past 63) or a block count
//       other than the interval's sets the image's status to B200_JPEG_ENTROPY_ERROR.
//    d. Each thread decodes its run once more from its exact entry state and writes its coefficients (de-zigzagged, into blocks
//       zeroed at the start); a segmented scan per component turns the DC differences into DC values.
//    Every read is bounded by the interval's length, every write by the interval's blocks.
// 2. jpeg_idct_kernel: dequantisation and libjpeg's islow IDCT (CONST_BITS 13, PASS1_BITS 2, 32-bit integers, range-limit
//    table), 8 threads per block (one column, then one row), into the component sample planes.
// 3. jpeg_color_kernel, one thread per output pixel: fancy upsampling of the chroma (libjpeg-turbo's h2v1 / h2v2 triangle
//    filters when the chroma row is wider than 2 samples, else replication; h1v2 always), the integer YCbCr -> BGR tables,
//    and the EXIF orientation, applied by reading the source pixel of each output pixel.
#include <cub/block/block_scan.cuh>

#include "common.cuh"

namespace b200 {

namespace {
constexpr int kHuffThreads = 1024;         // one CTA per interval: enough warps to cover the decode's latency chain
constexpr int kIdctThreads = 256;           // 32 blocks of 8 threads
constexpr int kColorThreads = 256;

struct St {                                 // a decoder state (in out[]: an exit state, cnt = 2 * blocks completed + error)
    int pos, blk, k, cnt;
};
__device__ __forceinline__ bool same(const St& a, const St& b) { return a.pos == b.pos && a.blk == b.blk && a.k == b.k; }
__device__ __forceinline__ St load_st(const int4* p) { const int4 v = *p; return St{v.x, v.y, v.z, v.w}; }
__device__ __forceinline__ void store_st(int4* p, const St& s) { *p = make_int4(s.pos, s.blk, s.k, s.cnt); }

// 32 bits of the interval starting at bit pos; bytes past the end read as 0
__device__ __forceinline__ unsigned window32(const unsigned char* __restrict__ d, int nbytes, int pos) {
    const int b = pos >> 3;
    unsigned long long x = 0;
#pragma unroll
    for (int i = 0; i < 5; ++i) x = (x << 8) | (b + i < nbytes ? (unsigned)__ldg(d + b + i) : 0u);
    return (unsigned)(x >> (8 - (pos & 7)));
}

// (length << 8) | symbol of the code at the front of the 16-bit window w; 0 for a bad code
__device__ __forceinline__ int huff_decode(const b200_jpeg_huff_table& t, unsigned w) {
    const int e = t.lookup[w >> (16 - 9)];
    if (e) return e;
    for (int l = 10; l <= 16; ++l) {
        const int c = (int)(w >> (16 - l));
        if (c <= t.maxcode[l]) return (l << 8) | t.values[c + t.valoff[l]];
    }
    return 0;
}

__device__ __forceinline__ int extend(unsigned v, int s) { return s && v < (1u << (s - 1)) ? (int)v - (1 << s) + 1 : (int)v; }

__constant__ unsigned char kZigzag[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// Decode from boundary state s up to the first boundary at or past `end` (oracle/jpeg.py decode_run).  Returns the exit state
// with cnt = 2 * blocks completed + error.  Data a valid stream never contains sets the error bit and the decode goes on, so
// that a decode from a guessed state can still fall into step with the true one: a bad code skips one bit, a code or magnitude
// past the interval ends it, a coefficient index past 63 ends the block.  With `out`, the n-th completed block goes to
// out + 64 * n while n < limit.
__device__ St decode_run(const unsigned char* __restrict__ d, int nbytes, St s, int end, const b200_jpeg_huff_table* dc,
                         const b200_jpeg_huff_table* ac, int hv, int bpm, short* __restrict__ out, int limit) {
    const int L = nbytes * 8;
    int n = 0, err = 0;
    while (s.pos < end) {
        const int rem = L - s.pos;
        const unsigned w = window32(d, nbytes, s.pos);
        if (s.k == 0 && rem < 8 && (w >> (32 - rem)) == (1u << rem) - 1u) {   // byte padding after the last block
            s.pos = L;
            break;
        }
        const int c = s.blk < hv ? 0 : s.blk - hv + 1;
        const int e = huff_decode(s.k == 0 ? dc[c] : ac[c], w >> 16);
        if (!e) {
            err = 1;
            s.pos += 1;
            continue;
        }
        const int ln = e >> 8, sym = e & 0xFF;
        bool done = false;
        if (s.k == 0) {
            if (ln + sym > rem) {
                err = 1;
                s.pos = L;
                break;
            }
            if (out && n < limit) out[64 * n] = (short)(sym ? extend((w << ln) >> (32 - sym), sym) : 0);
            s.pos += ln + sym;
            s.k = 1;
            continue;
        }
        const int r = sym >> 4, sz = sym & 15;
        if (sz) {
            if (ln + sz > rem) {
                err = 1;
                s.pos = L;
                break;
            }
            s.pos += ln + sz;
            s.k += r;
            if (s.k > 63) {
                err = 1;
                done = true;
            } else {
                if (out && n < limit) out[64 * n + kZigzag[s.k]] = (short)extend((w << ln) >> (32 - sz), sz);
                done = ++s.k == 64;
            }
        } else if (r == 15) {
            if (ln > rem) {
                err = 1;
                s.pos = L;
                break;
            }
            s.pos += ln;
            s.k += 16;
            done = s.k > 63;
            err |= done;
        } else {
            if (ln > rem) {
                err = 1;
                s.pos = L;
                break;
            }
            s.pos += ln;
            done = true;                                                        // EOB
        }
        if (done) {
            ++n;
            s.blk = s.blk + 1 < bpm ? s.blk + 1 : 0;
            s.k = 0;
        }
    }
    s.cnt = 2 * n + err;
    return s;
}

struct JpegWork {
    short* coef;              // (total_blocks, 64), blocks in MCU order per image
    unsigned char* planes;    // total_blocks * 64 samples
    int4* st_in;              // per subsequence
    int4* st_out;
};

__global__ void __launch_bounds__(kHuffThreads)
jpeg_huffman_kernel(const unsigned char* __restrict__ data, const b200_jpeg_desc* __restrict__ descs,
                    const b200_jpeg_interval* __restrict__ ivs, const b200_jpeg_huff_table* __restrict__ tables, int S, JpegWork w,
                    unsigned char* __restrict__ status) {
    using Scan = cub::BlockScan<int, kHuffThreads>;
    __shared__ b200_jpeg_huff_table tab[6];
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ int carry;
    const b200_jpeg_interval iv = ivs[blockIdx.x];
    const b200_jpeg_desc& D = descs[iv.image];
    const int nc = D.ncomp, hv = D.h * D.v, bpm = hv + (nc == 3 ? 2 : 0);
    {   // DC tables of the components, then their AC tables
        const int4* src = reinterpret_cast<const int4*>(tables + D.table);
        int4* dst = reinterpret_cast<int4*>(tab);
        const int n = 2 * nc * (int)(sizeof(b200_jpeg_huff_table) / 16);
        for (int i = threadIdx.x; i < n; i += kHuffThreads) dst[i] = __ldg(src + i);
    }
    const b200_jpeg_huff_table* dc = tab;
    const b200_jpeg_huff_table* ac = tab + nc;
    const int want = iv.num_mcus * bpm;
    short* coef = w.coef + 64 * (D.first_block + (long long)iv.first_mcu * bpm);
    {   // zero the interval's blocks
        int4* z = reinterpret_cast<int4*>(coef);
        for (long long i = threadIdx.x; i < 8LL * want; i += kHuffThreads) z[i] = make_int4(0, 0, 0, 0);
    }
    __syncthreads();
    const unsigned char* d = data + iv.data_offset;
    const int nbytes = iv.nbytes, L = 8 * nbytes;
    const int nsub = max(1, (int)(((long long)L + S - 1) / S));
    const int R = (nsub + kHuffThreads - 1) / kHuffThreads;
    const int j0 = min(nsub, threadIdx.x * R), j1 = min(nsub, j0 + R);
    int4* st_in = w.st_in + iv.first_subseq;
    int4* st_out = w.st_out + iv.first_subseq;
    auto sub_end = [&](int j) { return (int)min((long long)(j + 1) * S, (long long)L); };
    // a. speculative decode of the run
    {
        St s{j0 == 0 ? 0 : (int)min((long long)j0 * S, (long long)L), 0, 0, 0};
        for (int j = j0; j < j1; ++j) {
            store_st(st_in + j, s);
            s = decode_run(d, nbytes, s, sub_end(j), dc, ac, hv, bpm, nullptr, 0);
            store_st(st_out + j, s);
        }
    }
    // b. sync passes
    for (;;) {
        __syncthreads();
        St cand{0, 0, 0, 0};
        bool stale = false;
        if (j0 < j1 && j0 > 0) {
            cand = load_st(st_out + j0 - 1);
            stale = !same(cand, load_st(st_in + j0));
        }
        __syncthreads();
        if (stale) {
            St s = cand;
            for (int j = j0; j < j1; ++j) {
                if (j > j0 && same(s, load_st(st_in + j))) break;
                store_st(st_in + j, s);
                s = decode_run(d, nbytes, s, sub_end(j), dc, ac, hv, bpm, nullptr, 0);
                store_st(st_out + j, s);
            }
        }
        if (!__syncthreads_or(stale)) break;
    }
    // c. block counts
    int mine = 0, bad = 0;
    for (int j = j0; j < j1; ++j) {
        const int cnt = st_out[j].w;
        mine += cnt >> 1;
        bad |= cnt & 1;
    }
    int first, total;
    Scan(scan_tmp).ExclusiveSum(mine, first, total);
    const St last = load_st(st_out + nsub - 1);
    if (__syncthreads_or(bad) || !(last.pos == L && last.blk == 0 && last.k == 0) || total != want) {
        if (threadIdx.x == 0) status[iv.image] = B200_JPEG_ENTROPY_ERROR;
        return;
    }
    // d. decode again and write
    if (j0 < j1) {
        St s = load_st(st_in + j0);
        for (int j = j0; j < j1; ++j) {
            s = decode_run(d, nbytes, s, sub_end(j), dc, ac, hv, bpm, coef + 64LL * first, want - first);
            first += s.cnt >> 1;
        }
    }
    __syncthreads();
    // DC differences -> values: per component an inclusive scan over its blocks in MCU order, 32-bit wrapping like libjpeg's
    // unsigned sum, stored as 16 bits
    for (int c = 0; c < nc; ++c) {
        const int nb = c == 0 ? hv : 1, off = c == 0 ? 0 : hv + c - 1;
        const int n = iv.num_mcus * nb;
        if (threadIdx.x == 0) carry = 0;
        __syncthreads();
        for (int base = 0; base < n; base += kHuffThreads) {
            const int i = base + threadIdx.x;
            const long long blk = i < n ? (long long)(i / nb) * bpm + off + i % nb : 0;
            const int v = i < n ? coef[64 * blk] : 0;
            int incl, agg;
            Scan(scan_tmp).InclusiveSum(v, incl, agg);
            const int c0 = carry;
            if (i < n) coef[64 * blk] = (short)(int)((unsigned)incl + (unsigned)c0);
            __syncthreads();
            if (threadIdx.x == 0) carry = (int)((unsigned)c0 + (unsigned)agg);
            __syncthreads();
        }
    }
}

// islow constants, CONST_BITS = 13
constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299, F1847 = 15137,
              F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

// one islow pass on 8 values, descaled by `shift` with rounding
__device__ __forceinline__ void idct8(const int* in, int* out, int shift) {
    int z2 = in[2], z3 = in[6];
    int z1 = (z2 + z3) * F0541;
    const int tmp2 = z1 + z3 * -F1847, tmp3 = z1 + z2 * F0765;
    const int tmp0 = (in[0] + in[4]) * 8192, tmp1 = (in[0] - in[4]) * 8192;
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    int t0 = in[7], t1 = in[5], t2 = in[3], t3 = in[1];
    z1 = t0 + t3;
    z2 = t1 + t2;
    z3 = t0 + t2;
    int z4 = t1 + t3;
    const int z5 = (z3 + z4) * F1175;
    t0 *= F0298;
    t1 *= F2053;
    t2 *= F3072;
    t3 *= F1501;
    z1 *= -F0899;
    z2 *= -F2562;
    z3 = z3 * -F1961 + z5;
    z4 = z4 * -F0390 + z5;
    t0 += z1 + z3;
    t1 += z2 + z4;
    t2 += z2 + z3;
    t3 += z1 + z4;
    const int r = 1 << (shift - 1);
    out[0] = (tmp10 + t3 + r) >> shift;
    out[7] = (tmp10 - t3 + r) >> shift;
    out[1] = (tmp11 + t2 + r) >> shift;
    out[6] = (tmp11 - t2 + r) >> shift;
    out[2] = (tmp12 + t1 + r) >> shift;
    out[5] = (tmp12 - t1 + r) >> shift;
    out[3] = (tmp13 + t0 + r) >> shift;
    out[4] = (tmp13 - t0 + r) >> shift;
}

// libjpeg's range-limit table: value + 128 as a signed 10-bit number, clamped
__device__ __forceinline__ unsigned range_limit(int x) { return (unsigned)min(max(((x + 128 + 512) & 1023) - 512, 0), 255); }

__global__ void __launch_bounds__(kIdctThreads)
jpeg_idct_kernel(const b200_jpeg_desc* __restrict__ descs, JpegWork w, const unsigned char* __restrict__ status) {
    __shared__ int ws[kIdctThreads / 8][8][8];
    const int img = blockIdx.y;
    if (status[img]) return;
    const b200_jpeg_desc& D = descs[img];
    const int nc = D.ncomp, hv = D.h * D.v, bpm = hv + (nc == 3 ? 2 : 0);
    const long long mcus = (long long)D.mcus_x * D.mcus_y, nblocks = mcus * bpm;
    const int slot = threadIdx.x >> 3, r = threadIdx.x & 7;
    unsigned char* planes = w.planes + 64 * D.first_block;
    for (long long b = (long long)blockIdx.x * (kIdctThreads / 8) + slot; b < nblocks; b += (long long)gridDim.x * (kIdctThreads / 8)) {
        const long long m = b / bpm;
        const int blk = (int)(b % bpm);
        const int c = blk < hv ? 0 : blk - hv + 1;
        const long long mx = m % D.mcus_x, my = m / D.mcus_x;
        const short* cf = w.coef + 64 * (D.first_block + b);
        const unsigned short* q = D.quant[c];
        int col[8], o[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) col[u] = (int)cf[8 * u + r] * (int)q[8 * u + r];
        idct8(col, o, 11);
#pragma unroll
        for (int u = 0; u < 8; ++u) ws[slot][u][r] = o[u];
        __syncwarp();
        int row[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) row[u] = ws[slot][r][u];
        idct8(row, o, 18);
        __syncwarp();
        long long pitch, y, x;
        unsigned char* plane;
        if (c == 0) {
            pitch = (long long)D.mcus_x * D.h * 8;
            y = (my * D.v + blk / D.h) * 8 + r;
            x = (mx * D.h + blk % D.h) * 8;
            plane = planes;
        } else {
            pitch = (long long)D.mcus_x * 8;
            y = my * 8 + r;
            x = mx * 8;
            plane = planes + 64 * mcus * hv + 64 * mcus * (c - 1);
        }
        uint2 v;
        v.x = range_limit(o[0]) | range_limit(o[1]) << 8 | range_limit(o[2]) << 16 | range_limit(o[3]) << 24;
        v.y = range_limit(o[4]) | range_limit(o[5]) << 8 | range_limit(o[6]) << 16 | range_limit(o[7]) << 24;
        *reinterpret_cast<uint2*>(plane + y * pitch + x) = v;
    }
}

// chroma sample of plane p (pitch, real size cw x ch) upsampled to luma position (y, x) for luma sampling h x v
__device__ __forceinline__ int chroma(const unsigned char* __restrict__ p, long long pitch, int cw, int ch, int h, int v, int y, int x) {
    if (h == 1 && v == 1) return p[(long long)y * pitch + x];
    if (h == 2 && cw <= 2) return p[(long long)(y >> (v - 1)) * pitch + (x >> 1)];   // replication
    if (h == 1) {                                                                     // h1v2
        const int i = y >> 1, odd = y & 1;
        const int nb = odd ? min(i + 1, ch - 1) : max(i - 1, 0);
        return (3 * p[(long long)i * pitch + x] + p[(long long)nb * pitch + x] + 1 + odd) >> 2;
    }
    const int j = x >> 1, right = x & 1;
    const int jn = right ? min(j + 1, cw - 1) : max(j - 1, 0);
    if (v == 1) {                                                                     // h2v1
        const unsigned char* row = p + (long long)y * pitch;
        return (3 * row[j] + row[jn] + 1 + right) >> 2;
    }
    const int i = y >> 1, odd = y & 1;                                                // h2v2
    const int in = odd ? min(i + 1, ch - 1) : max(i - 1, 0);
    const unsigned char* r0 = p + (long long)i * pitch;
    const unsigned char* r1 = p + (long long)in * pitch;
    const int s = 3 * r0[j] + r1[j], sn = 3 * r0[jn] + r1[jn];
    return (3 * s + sn + 8 - right) >> 4;
}

__global__ void __launch_bounds__(kColorThreads)
jpeg_color_kernel(const b200_jpeg_desc* __restrict__ descs, JpegWork w, const unsigned char* __restrict__ status,
                  unsigned char* __restrict__ out) {
    const int img = blockIdx.y;
    if (status[img]) return;
    const b200_jpeg_desc& D = descs[img];
    const int H = D.height, W = D.width, o = D.orientation;
    const int OW = o >= 5 ? H : W;
    const long long n = (long long)H * W;
    const long long mcus = (long long)D.mcus_x * D.mcus_y;
    const unsigned char* y_plane = w.planes + 64 * D.first_block;
    const long long ypitch = (long long)D.mcus_x * D.h * 8, cpitch = (long long)D.mcus_x * 8;
    const unsigned char* cb_plane = y_plane + 64 * mcus * D.h * D.v;
    const unsigned char* cr_plane = cb_plane + 64 * mcus;
    const int cw = (W + D.h - 1) / D.h, ch = (H + D.v - 1) / D.v;
    unsigned char* dst = out + D.out_offset;
    for (long long t = (long long)blockIdx.x * kColorThreads + threadIdx.x; t < n; t += (long long)gridDim.x * kColorThreads) {
        const int oy = (int)(t / OW), ox = (int)(t % OW);
        int sy, sx;
        switch (o) {
            case 2: sy = oy; sx = W - 1 - ox; break;
            case 3: sy = H - 1 - oy; sx = W - 1 - ox; break;
            case 4: sy = H - 1 - oy; sx = ox; break;
            case 5: sy = ox; sx = oy; break;
            case 6: sy = H - 1 - ox; sx = oy; break;
            case 7: sy = H - 1 - ox; sx = W - 1 - oy; break;
            case 8: sy = ox; sx = W - 1 - oy; break;
            default: sy = oy; sx = ox; break;
        }
        const int Y = y_plane[(long long)sy * ypitch + sx];
        int b = Y, g = Y, r = Y;
        if (D.ncomp == 3) {
            const int cb = chroma(cb_plane, cpitch, cw, ch, D.h, D.v, sy, sx) - 128;
            const int cr = chroma(cr_plane, cpitch, cw, ch, D.h, D.v, sy, sx) - 128;
            r = Y + ((91881 * cr + 32768) >> 16);
            g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
            b = Y + ((116130 * cb + 32768) >> 16);
        }
        unsigned char* px = dst + 3 * t;
        px[0] = (unsigned char)min(max(b, 0), 255);
        px[1] = (unsigned char)min(max(g, 0), 255);
        px[2] = (unsigned char)min(max(r, 0), 255);
    }
}

size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }
}  // namespace

}  // namespace b200

using namespace b200;

extern "C" {

size_t b200_jpeg_decode_workspace_bytes(long long total_blocks, long long total_subseqs) {
    if (total_blocks < 1 || total_subseqs < 1) return 0;
    return align_up((size_t)total_blocks * 128) + align_up((size_t)total_blocks * 64) + 2 * align_up((size_t)total_subseqs * 16);
}

int b200_jpeg_decode(const unsigned char* data_dev, const b200_jpeg_desc* descs_dev, int num_images, const b200_jpeg_interval* intervals_dev,
                     int num_intervals, const b200_jpeg_huff_table* tables_dev, int subseq_bits, long long total_blocks,
                     long long total_subseqs, long long max_blocks, long long max_pixels, void* workspace, size_t workspace_bytes,
                     unsigned char* out_dev, unsigned char* status_dev, b200_stream_t stream) {
    if (!data_dev || !descs_dev || !intervals_dev || !tables_dev || !workspace || !out_dev || !status_dev) return B200_ROI_EINVAL;
    if (num_images < 1 || num_images > 65535 || num_intervals < num_images || subseq_bits < 1 || total_blocks < 1 || total_subseqs < 1 ||
        max_blocks < 1 || max_blocks > total_blocks || max_pixels < 1)
        return B200_ROI_EINVAL;
    if (workspace_bytes < b200_jpeg_decode_workspace_bytes(total_blocks, total_subseqs)) return B200_ROI_EWORKSPACE;
    char* ws = static_cast<char*>(workspace);
    JpegWork w;
    w.coef = reinterpret_cast<short*>(ws);
    ws += align_up((size_t)total_blocks * 128);
    w.planes = reinterpret_cast<unsigned char*>(ws);
    ws += align_up((size_t)total_blocks * 64);
    w.st_in = reinterpret_cast<int4*>(ws);
    ws += align_up((size_t)total_subseqs * 16);
    w.st_out = reinterpret_cast<int4*>(ws);
    cudaMemsetAsync(status_dev, 0, (size_t)num_images, stream);
    jpeg_huffman_kernel<<<num_intervals, kHuffThreads, 0, stream>>>(data_dev, descs_dev, intervals_dev, tables_dev, subseq_bits, w,
                                                                    status_dev);
    const unsigned idct_x = (unsigned)min((max_blocks + kIdctThreads / 8 - 1) / (kIdctThreads / 8), 1LL << 20);
    jpeg_idct_kernel<<<dim3(idct_x, num_images), kIdctThreads, 0, stream>>>(descs_dev, w, status_dev);
    const unsigned color_x = (unsigned)min((max_pixels + kColorThreads - 1) / kColorThreads, 1LL << 20);
    jpeg_color_kernel<<<dim3(color_x, num_images), kColorThreads, 0, stream>>>(descs_dev, w, status_dev, out_dev);
    return finish_launch(3);
}

}  // extern "C"
