// Kernel Audio Distance (KAD): Gaussian-kernel MMD between two embedding sets on Hopper tensor cores (wgmma).
//
// Z = [X; Y] (fp16 [N = m + n, d], X first).  Every pair i < j of rows of Z is one of: an xx pair, a yy pair, or an xy
// pair, each exactly once, so ONE pass over the upper-triangular 128 x 128 tiles of Z Z^T yields
//   S_xx = sum_{i<j<m} k(z_i, z_j),  S_yy = sum_{m<=i<j} k(z_i, z_j),  S_xy = sum_{i<m<=j} k(z_i, z_j),
//   k(a, b) = exp(-|a - b|^2 / (2 sigma^2)).
//
// The distances, the prologue (shift, hi/lo split, row norms), the tile loop and the warp roles are the pair-tile code
// both pairwise metrics run (pair_tile.cuh); this file holds what KAD alone runs: the tile kernel's three epilogues
// (q, ex2 or histogram, masks, class sums) and the reductions and selection after it.
//
// Work units and determinism.  T = ceil(N / 128) tile rows; unit u (u < ceil(T / 2)) is tile row u (tiles u..T-1)
// followed by tile row T-1-u (tiles T-1-u..T-1): T + 1 tiles per unit, so units are balanced.  A launch covers the
// units [unit0, unit1) (all of them, or one shard of a sharded call), and a CTA takes units unit0 + blockIdx.x,
// + gridDim.x, ...  Each consumer thread sums its elements of a tile in fp32 (fixed order), adds that to
// fp64 per-thread accumulators in tile order, and at the end of the unit the 256 consumer threads are reduced in a
// fixed tree into partial[u][3] (fp64).  kad_reduce_kernel sums the partials in unit order.  No floating-point atomic
// anywhere: the three sums are bitwise reproducible and independent of the grid size and of timing.
//
// Per-song sums (MODE 2).  Z = [X; Y_1; ...; Y_K]; S_xx comes from MODE 0 over the first m rows.  The A operand is a
// 128-row tile of Y (rows m + 128 t, not tile-aligned in Z); the B operands are the X tiles (mask j < m), then the
// song band: Y tiles t .. the tile holding the last row of the song that owns tile t's last row (mask i < j < end of
// i's song, read from song_of and offsets as the per-song PRDC passes read them).  Work unit = (Y tile, up to G
// consecutive column tiles), G a function of the shape only (host work list).  Each thread sums k over its columns per
// row in fp32 per tile and in fp64 over the unit's tiles; the quad's 4 lanes are added by a fixed shuffle tree into
// partial[u][row] (S_xy and S_yy).  kad_song_reduce_kernel adds each row's units in order, then each song's rows in a
// fixed tree: no atomics, bitwise reproducible, independent of the grid.
//
// Bandwidth (MODE 1): exact selection of the two middle q values of the xx triangle by radix passes over the fp32 bit
// pattern of q (monotone for q >= 0): bits 30..20, 19..10, 9..0.  Each pass runs the same tile loop over X alone and
// counts the q values whose already-selected high bits match each of the two targets into shared-memory histograms,
// flushed into 64-bit global counts with integer atomics (order-independent); kad_select_kernel picks the bin of each
// target.  The q values are bit-for-bit the ones the sums kernel computes for the same rows.
#pragma once
#include "pair_tile.cuh"

namespace fad {

constexpr int kKadHistBins = 2048;                  // per target; the largest radix digit has 11 bits
constexpr uint32_t kKadHistBytes = 2 * kKadHistBins * 4;
constexpr uint32_t kKadSmemBytes = kPairSmemBytes + 256 /*unit reduction*/ + kKadHistBytes;
static_assert(kKadSmemBytes <= 227 * 1024, "over the per-CTA shared-memory limit");

struct KadParams {
    int N;                   // rows of Z (X rows first)
    int m;                   // rows of X
    int d;                   // columns
    int T;                   // tile rows = ceil(N / 128)
    int units;               // ceil(T / 2) (MODE 2: the work list's length)
    int unit0, unit1;        // this launch's units [unit0, unit1) (a shard; partials stay indexed by the global unit)
    const float* norm;       // [T * 128] |y_i|^2 (zero past N; MODE 2: [m + Ty * 128])
    // MODE 0 and 2
    const double* sigma;     // device scalar
    double* partial;         // MODE 0: [units][3]; MODE 2: [units][2][128] per-row S_xy, S_yy
    // MODE 1
    const uint32_t* prefix;  // [2] selected high bits of the two targets
    unsigned long long* hist;// [2][kKadHistBins] global counts
    uint32_t mask;           // bits already selected
    int shift, bins;         // digit of this pass: (u >> shift) & (bins - 1)
    // MODE 2 (per-song sums): A = a 128-row tile of Y (rows m + 128 t ...), B = the tiles of X, then the song band
    const int4* work;        // [units] {t, v0, v1}: virtual column tiles [v0, v1) of Y tile t; v < Tx: X tile v,
                             // v >= Tx: Y tile t + v - Tx
    const int* song_of;      // [Ty * 128] the song of each Y row, -1 past the last row (pair_song_of_kernel)
    const long long* offsets;// [songs + 1] song s = Y rows [offsets[s], offsets[s + 1])
    int Tx;                  // ceil(m / 128)
};

template <int MODE>
__global__ void __launch_bounds__(kPairThreads, 1)
kad_tile_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo, const KadParams p) {
    using namespace sm90;
    static_assert(MODE == 0 || MODE == 1 || MODE == 2, "0: kernel sums, 1: radix histogram of q, 2: per-row song sums");
    extern __shared__ uint8_t smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const PairTile pt = pair_tile_open(smem_raw, &map_hi, &map_lo, p.d, warp, lane);
    uint8_t* smem = pt.smem;
    uint64_t* full = pt.full;
    uint64_t* empty = pt.empty;
    const int ksteps = pt.ksteps, chunk_len = pt.chunk_len;
    double* red = reinterpret_cast<double*>(pt.own);                // [8 warps][3]
    uint32_t* hist = reinterpret_cast<uint32_t*>(pt.own + 256);     // [2][kKadHistBins]
    if (MODE == 1)
        for (int b = threadIdx.x; b < 2 * kKadHistBins; b += kPairThreads) hist[b] = 0;
    __syncthreads();

    if (warp < 4) {
        // ------------------------------------------------------------ TMA producer
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            int s = 0; uint32_t ph = 0;
            if constexpr (MODE == 2) {
                for (int u = p.unit0 + blockIdx.x; u < p.unit1; u += gridDim.x) {
                    const int4 wk = p.work[u];
                    const int arow = p.m + wk.x * 128;
                    for (int v = wk.y; v < wk.z; ++v)
                        pair_load_tile(smem, full, empty, s, ph, &map_hi, &map_lo, ksteps, arow,
                                       v < p.Tx ? v * 128 : arow + (v - p.Tx) * 128);
                }
            } else {
                for (int u = p.unit0 + blockIdx.x; u < p.unit1; u += gridDim.x) {
                    for (int half = 0; half < 2; ++half) {
                        const int r = half == 0 ? u : p.T - 1 - u;
                        if (half == 1 && r == u) break;                // odd T: the middle row once
                        for (int ct = r; ct < p.T; ++ct)
                            pair_load_tile(smem, full, empty, s, ph, &map_hi, &map_lo, ksteps, r * 128, ct * 128);
                    }
                }
            }
        }
    } else {
        // ------------------------------------------------------------ consumers: wgmma + epilogue in registers
        setmaxnreg_inc<kPairConsumerRegs>();
        const int c = (warp >> 2) - 1;                    // tile rows [64 c, 64 c + 64)
        const int wq = warp & 3;
        const int ct_id = threadIdx.x - 128;              // 0..255
        int s = 0; uint32_t ph = 0;
        if constexpr (MODE == 2) {
            const double sg = *p.sigma;
            const float neg_coef = (float)(-1.4426950408889634 / (2.0 * sg * sg));
            const int lr0 = c * 64 + wq * 16 + (lane >> 2);                    // tile rows lr0, lr0 + 8
            for (int u = p.unit0 + blockIdx.x; u < p.unit1; u += gridDim.x) {
                const int4 wk = p.work[u];
                const int row0 = p.m + wk.x * 128 + lr0;                       // rows of Z
                const float nr[2] = {__ldg(p.norm + row0), __ldg(p.norm + row0 + 8)};
                // the end row (in Z) of each row's song; 0 past the last row
                int end[2];
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int sg = __ldg(p.song_of + row0 + 8 * i - p.m);
                    end[i] = sg < 0 ? 0 : p.m + (int)__ldg(p.offsets + sg + 1);
                }
                double axy[2] = {0.0, 0.0}, ayy[2] = {0.0, 0.0};
                for (int v = wk.y; v < wk.z; ++v) {
                    const bool xt = v < p.Tx;
                    const int col0 = (xt ? v * 128 : p.m + (wk.x + v - p.Tx) * 128) + 2 * (lane & 3);
                    // columns j of row i that count: X tile j < m (none for a row past the last song, end = 0);
                    // band tile i < j < end of the song of row i
                    int lo[2], hi[2];
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        lo[i] = xt ? -1 : row0 + 8 * i;
                        hi[i] = xt ? (end[i] > 0 ? p.m : 0) : end[i];
                    }
                    float sum[64];
                    pair_mma_tile(sum, smem, full, empty, s, ph, c, lane, p.d, ksteps, chunk_len);
                    float rs[2] = {0.f, 0.f};
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        // col0 has the parity of m in band tiles: two scalar loads, not a float2
                        const float nc[2] = {__ldg(p.norm + col0 + 8 * j), __ldg(p.norm + col0 + 8 * j + 1)};
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int gj = col0 + 8 * j + e;
                                const float q = pair_q(sum[4 * j + 2 * i + e], nr[i], nc[e]);
                                float kv;
                                asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(kv) : "f"(q * neg_coef));
                                rs[i] += (gj > lo[i] && gj < hi[i]) ? kv : 0.f;
                            }
                        }
                    }
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        if (xt) axy[i] += (double)rs[i]; else ayy[i] += (double)rs[i];
                    }
                }
                // the 4 lanes of a quad hold the same two rows: fixed xor tree, then one lane writes each row
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    for (int o = 1; o < 4; o <<= 1) {
                        axy[i] += __shfl_xor_sync(0xffffffffu, axy[i], o);
                        ayy[i] += __shfl_xor_sync(0xffffffffu, ayy[i], o);
                    }
                    if ((lane & 3) == 0) {
                        p.partial[(size_t)u * 256 + lr0 + 8 * i] = axy[i];
                        p.partial[(size_t)u * 256 + 128 + lr0 + 8 * i] = ayy[i];
                    }
                }
            }
            return;
        }
        float neg_coef = 0.f;
        uint32_t pfx0 = 0, pfx1 = 0;
        bool two = false;
        if (MODE == 0) {
            const double sg = *p.sigma;
            neg_coef = (float)(-1.4426950408889634 / (2.0 * sg * sg));
        } else {
            pfx0 = p.prefix[0]; pfx1 = p.prefix[1];
            two = pfx0 != pfx1;
        }
        const uint32_t digit_mask = (uint32_t)p.bins - 1;

        for (int u = p.unit0 + blockIdx.x; u < p.unit1; u += gridDim.x) {
            double sxx = 0.0, syy = 0.0, sxy = 0.0;
            for (int half = 0; half < 2; ++half) {
                const int r = half == 0 ? u : p.T - 1 - u;
                if (half == 1 && r == u) break;
                const int row0 = r * 128 + c * 64 + wq * 16 + (lane >> 2);     // rows row0, row0 + 8
                const float nr0 = __ldg(p.norm + row0), nr1 = __ldg(p.norm + row0 + 8);
                for (int ct = r; ct < p.T; ++ct) {
                    float sum[64];
                    pair_mma_tile(sum, smem, full, empty, s, ph, c, lane, p.d, ksteps, chunk_len);

                    // ---- epilogue on the fragment: element (row0 + 8 i, col0 + 8 j + e) is sum[4 j + 2 i + e]
                    const int col0 = ct * 128 + 2 * (lane & 3);
                    float sx[2] = {0.f, 0.f}, sy[2] = {0.f, 0.f};
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const float2 nc = __ldg(reinterpret_cast<const float2*>(p.norm + col0 + 8 * j));
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const int gi = row0 + 8 * i, gj = col0 + 8 * j + e;
                                const float q = pair_q(sum[4 * j + 2 * i + e], i ? nr1 : nr0, e ? nc.y : nc.x);
                                const bool valid = gj > gi && gj < p.N;        // index masks: j > i, no zero-filled row
                                if (MODE == 0) {
                                    float kv;
                                    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(kv) : "f"(q * neg_coef));
                                    kv = valid ? kv : 0.f;
                                    if (gj < p.m) sx[i] += kv; else sy[i] += kv;
                                } else if (valid) {
                                    const uint32_t bits = __float_as_uint(q);
                                    const uint32_t bin = (bits >> p.shift) & digit_mask;
                                    if ((bits & p.mask) == pfx0) atomicAdd(&hist[bin], 1u);
                                    else if (two && (bits & p.mask) == pfx1) atomicAdd(&hist[kKadHistBins + bin], 1u);
                                }
                            }
                        }
                    }
                    if (MODE == 0) {
                        // j > i: a row of Y pairs only with rows of Y
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            if (row0 + 8 * i < p.m) { sxx += (double)sx[i]; sxy += (double)sy[i]; }
                            else syy += (double)sy[i];
                        }
                    }
                }
            }

            if (MODE == 0) {
                // fixed tree: lanes (shuffle), then the 8 consumer warps in order
                for (int o = 16; o > 0; o >>= 1) {
                    sxx += __shfl_xor_sync(0xffffffffu, sxx, o);
                    syy += __shfl_xor_sync(0xffffffffu, syy, o);
                    sxy += __shfl_xor_sync(0xffffffffu, sxy, o);
                }
                const int cw = ct_id >> 5;
                if (lane == 0) { red[cw * 3 + 0] = sxx; red[cw * 3 + 1] = syy; red[cw * 3 + 2] = sxy; }
                named_bar_sync(1, 256);
                if (ct_id < 3) {
                    double t = 0.0;
                    for (int w = 0; w < 8; ++w) t += red[w * 3 + ct_id];
                    p.partial[(size_t)u * 3 + ct_id] = t;
                }
                named_bar_sync(1, 256);
            } else {
                // per unit, so a CTA's 32-bit bins cannot overflow (a unit has (T + 1) x 16384 elements)
                named_bar_sync(1, 256);
                for (int b = ct_id; b < 2 * kKadHistBins; b += 256) {
                    const uint32_t v = hist[b];
                    if (v) { atomicAdd(p.hist + b, (unsigned long long)v); hist[b] = 0; }
                }
                named_bar_sync(1, 256);
            }
        }
    }
}

// --------------------------------------------------------------------------------------------- epilogues
// out[t] = sum over units, in unit order, of partial[u][t]
__global__ void kad_reduce_kernel(const double* __restrict__ partial, int units, double* __restrict__ out) {
    const int t = threadIdx.x;
    if (t >= 3) return;
    double s = 0.0;
    for (int u = 0; u < units; ++u) s += partial[(size_t)u * 3 + t];
    out[t] = s;
}

// one block per song: out[2k] = S_yy,k, out[2k + 1] = S_xy,k.  Each row's partials are summed over the units of its
// tile in unit order, a thread's rows in row order, then the block in a fixed tree - a fixed order for a given shape.
constexpr int kKadSongReduceThreads = 128;
__global__ void __launch_bounds__(kKadSongReduceThreads)
kad_song_reduce_kernel(const double* __restrict__ partial, const int* __restrict__ unit_start,
                       const long long* __restrict__ offsets, double* __restrict__ out) {
    __shared__ double red[2][kKadSongReduceThreads / 32];
    const int k = blockIdx.x;
    double xy = 0.0, yy = 0.0;
    for (long long r = offsets[k] + threadIdx.x; r < offsets[k + 1]; r += kKadSongReduceThreads) {
        const int t = (int)(r >> 7), lr = (int)(r & 127);
        double rx = 0.0, ry = 0.0;
        for (int u = unit_start[t]; u < unit_start[t + 1]; ++u) {
            rx += partial[(size_t)u * 256 + lr];
            ry += partial[(size_t)u * 256 + 128 + lr];
        }
        xy += rx;
        yy += ry;
    }
    for (int o = 16; o > 0; o >>= 1) {
        xy += __shfl_xor_sync(0xffffffffu, xy, o);
        yy += __shfl_xor_sync(0xffffffffu, yy, o);
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { red[0][w] = xy; red[1][w] = yy; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double sxy = 0.0, syy = 0.0;
        for (int i = 0; i < kKadSongReduceThreads / 32; ++i) { sxy += red[0][i]; syy += red[1][i]; }
        out[2 * (size_t)k] = syy;
        out[2 * (size_t)k + 1] = sxy;
    }
}

// state: prefix[2] (u32), then rank[2] (u64) = the rank of each target among the values that match its prefix
struct KadSelectState {
    uint32_t prefix[2];
    unsigned long long rank[2];
};
__global__ void kad_select_init_kernel(KadSelectState* st, unsigned long long k0, unsigned long long k1) {
    st->prefix[0] = st->prefix[1] = 0u;
    st->rank[0] = k0;
    st->rank[1] = k1;
}
// after a histogram pass: the bin of each target's rank; when both targets still shared a prefix, the pass counted
// into histogram 0 only.  last: write the two selected q values (fp64) to out.
__global__ void kad_select_kernel(KadSelectState* st, const unsigned long long* __restrict__ hist, int shift, int bins,
                                  int last, double* __restrict__ out) {
    if (threadIdx.x != 0) return;
    const bool two = st->prefix[0] != st->prefix[1];
    for (int t = 0; t < 2; ++t) {
        const unsigned long long* h = hist + (two ? t : 0) * kKadHistBins;
        unsigned long long r = st->rank[t], below = 0;
        int b = 0;
        for (; b < bins - 1; ++b) {
            if (below + h[b] > r) break;
            below += h[b];
        }
        st->prefix[t] |= (uint32_t)b << shift;
        st->rank[t] = r - below;
    }
    if (last) {
        out[0] = (double)__uint_as_float(st->prefix[0]);
        out[1] = (double)__uint_as_float(st->prefix[1]);
    }
}

// ------------------------------------------------------------------------------- permutation tests (DESIGN.md 5.16)
// Z = a pool of N rows; a labelling marks `a` of them.  Over the pairs i < j, with K_ij the kernel value rounded to fp16
// once: R_i = sum_{j>i} K_ij, P(l) = sum l_i l_j K_ij, C(l) = sum l_j K_ij.  The tile pass runs MODE 0's units and tiles;
// each consumer stores its 64 x 128 block of fp16 kernel values to shared memory (K-major, 128-B swizzle) and runs, per
// block of 64 labellings, U = W_J K_IJ^T as 8 m64n64k16 wgmmas with the labels of the column tile J expanded from bits
// to fp16 0 / 1 in registers (the A operand).  The accumulator holds (labelling, row i); each thread sums its elements
// over i in fp32 (C) and over the rows of I the labelling marks (P), a fixed quad tree adds the 4 lanes of a labelling,
// and each lane keeps one fp64 running sum per block over the unit's tiles.  R_i is summed per thread over the unit's
// tiles in fp64 and written once (a tile row belongs to one unit).  No atomics: every sum has a fixed order.
//
// Label bits: labelling b is words [b * words, (b + 1) * words), words = 4 ceil(N / 128); bit i & 31 of word i >> 5 is
// row i's label, 0 past N.  Labelling 0 marks rows 0 .. a - 1; labelling b >= 1 marks the a rows with the smallest
// (pair_mix64(pair_mix64(seed + b) ^ i), i); labellings past the last are all zero.
//
// kBoot (the bootstrap, DESIGN.md 5.18): Q(v) = sum_{i<j} v_i v_j K_ij for row weights v (resamples in place of
// labellings, the fp16 integer weights [rows][T * 128] in place of the bits; exact up to 2048).  The A operand is the
// column tile's weights, the reduction over i multiplies by v_i, the shrink is undone counting the nonzero-weight
// columns, and C and R are not formed (C's partial slots are written as 0).
constexpr int kPermBlock = 64;                     // labellings per wgmma (its M)
constexpr int kPermPass = 1024;                    // labellings per tile pass
constexpr int kPermLabelThreads = 1024;
constexpr int kPermSumThreads = 256;
constexpr uint32_t kPermKBytes = 64 * 128 * 2;     // one consumer's fp16 kernel block: two 64-row x 64-column halves
// the pair tiles, then (1024-aligned: 768 bytes past the barriers) the two consumers' kernel blocks
constexpr uint32_t kPermSmemBytes = kPairSmemBytes + 768 + 2 * kPermKBytes;
static_assert(kPermSmemBytes <= 227 * 1024, "over the per-CTA shared-memory limit");

struct KadPermParams {
    int N, d, T;
    int units, unit0, unit1;  // MODE 0's units; this launch's [unit0, unit1)
    const float* norm;        // [T * 128]
    const double* sigma;      // device scalar
    const uint32_t* bits;     // this pass's first labelling (layout above)
    int words;                // words per labelling
    int blocks;               // blocks of 64 labellings in this pass (1 .. 16)
    double* partial;          // [units][2 consumers][64 blocks][2]: P, C of each labelling
    double* rowsum;           // [T * 128] R_i
    const __half* weights;    // kBoot: this pass's first resample's row weights [rows][T * 128] (bits, rowsum unused)
};

// bits b0, b1 (bits 0, 1 of x) -> the fp16 pair (b0, b1) as 0 / 1
__device__ __forceinline__ uint32_t perm_half2(uint32_t x) {
    return ((x & 1u) | ((x & 2u) << 15)) * 0x3C00u;
}

// kBoot's label product of one column tile ct of tile row r: per block of 64 resamples, U = V_J K_IJ^T as the 8
// wgmmas of the labellings with the weights of J as the A operand, then P = sum_i v_i U_i over the rows of I, added to
// acc[block] with the shrink of the columns of J whose weight is nonzero undone.  The weight rows are advanced through
// an empty asm as the bits are.
__device__ __forceinline__ void boot_label_product(double (&acc)[kPermPass / kPermBlock], const KadPermParams& p,
                                                   uint32_t kbase, int lr0, int q, int c, int r, int ct) {
    using namespace sm90;
    const size_t stride = (size_t)p.T * 64;                     // words (fp16 pairs) per resample row
    const uint32_t* wl = reinterpret_cast<const uint32_t*>(p.weights) + (size_t)lr0 * stride;
    const size_t row8 = 8 * stride, block = (size_t)kPermBlock * stride;
#pragma unroll
    for (int lb = 0; lb < kPermPass / kPermBlock; ++lb) {
        if (lb < p.blocks) {
            // A fragment of k-step kk: a[0] = resample row lr0, columns 16 kk + 2 q + {0, 1}; a[1] = row lr0 + 8;
            // a[2], a[3] = columns + 8
            const uint32_t* wj = wl + ct * 64 + q;
            uint32_t a[8][4];
            int nz[2] = {0, 0};
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                a[kk][0] = __ldg(wj + 8 * kk);
                a[kk][1] = __ldg(wj + row8 + 8 * kk);
                a[kk][2] = __ldg(wj + 8 * kk + 4);
                a[kk][3] = __ldg(wj + row8 + 8 * kk + 4);
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    nz[e & 1] += ((a[kk][e] & 0xFFFFu) != 0u) + ((a[kk][e] >> 16) != 0u);
            }
            float dl[32];
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk)
                wgmma_m64n64k16_f16_rs_kmajor(dl, a[kk], kmajor_sw128_desc(kbase + (kk >> 2) * (kPermKBytes / 2)) + 2 * (kk & 3),
                                              kk > 0);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(dl);
            // element (resample row lr0 + 8 rr, row 64 c + 8 jj + 2 q + e of I) is dl[4 jj + 2 rr + e]; its weight is
            // half e of word r * 64 + 32 c + 4 jj + q of the resample row
            const uint32_t* wi = wl + r * 64 + 32 * c + q;
            float pp[2] = {0.f, 0.f};
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    const uint32_t w = __ldg(wi + (rr ? row8 : 0) + 4 * jj);
                    pp[rr] = fmaf(dl[4 * jj + 2 * rr], __half2float(__ushort_as_half((unsigned short)(w & 0xFFFFu))), pp[rr]);
                    pp[rr] = fmaf(dl[4 * jj + 2 * rr + 1], __half2float(__ushort_as_half((unsigned short)(w >> 16))), pp[rr]);
                }
            }
#pragma unroll
            for (int o = 1; o < 4; o <<= 1) {
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    pp[rr] += __shfl_xor_sync(0xffffffffu, pp[rr], o);
                    nz[rr] += __shfl_xor_sync(0xffffffffu, nz[rr], o);
                }
            }
            // lane q keeps P of resample row lr0 + 8 (q >> 1) (q even; odd lanes add 0 to C's slot); the shrink is undone
            // as in the labelled pass, counting the columns of J with a nonzero weight
            const float mine = q == 0 ? pp[0] : q == 2 ? pp[1] : 0.f;
            const int marked = q < 2 ? nz[0] : nz[1];
            acc[lb] += (double)fmaf(mine, kAccumShrinkPerElement * (float)marked, mine);
            wl += block;
            asm volatile("" : "+l"(wl));
        }
    }
}

template <bool kBoot>
__global__ void __launch_bounds__(kPairThreads, 1)
kad_perm_tile_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                     const KadPermParams p) {
    using namespace sm90;
    extern __shared__ uint8_t smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const PairTile pt = pair_tile_open(smem_raw, &map_hi, &map_lo, p.d, warp, lane);
    uint8_t* smem = pt.smem;
    uint64_t* full = pt.full;
    uint64_t* empty = pt.empty;
    const int ksteps = pt.ksteps, chunk_len = pt.chunk_len;
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            int s = 0; uint32_t ph = 0;
            for (int u = p.unit0 + blockIdx.x; u < p.unit1; u += gridDim.x) {
                for (int half = 0; half < 2; ++half) {
                    const int r = half == 0 ? u : p.T - 1 - u;
                    if (half == 1 && r == u) break;
                    for (int ct = r; ct < p.T; ++ct)
                        pair_load_tile(smem, full, empty, s, ph, &map_hi, &map_lo, ksteps, r * 128, ct * 128);
                }
            }
        }
        return;
    }
    setmaxnreg_inc<kPairConsumerRegs>();
    const int c = (warp >> 2) - 1;
    const int wq = warp & 3;
    const int q = lane & 3;
    const int lr0 = wq * 16 + (lane >> 2);        // rows lr0, lr0 + 8 of the consumer's 64; also labelling rows of a block
    const uint32_t kbase = smem_u32(pt.own + 768) + c * kPermKBytes;
    const double sg = *p.sigma;
    const float neg_coef = (float)(-1.4426950408889634 / (2.0 * sg * sg));
    int s = 0; uint32_t ph = 0;

    for (int u = p.unit0 + blockIdx.x; u < p.unit1; u += gridDim.x) {
        double acc[kPermPass / kPermBlock];
#pragma unroll
        for (int lb = 0; lb < kPermPass / kPermBlock; ++lb) acc[lb] = 0.0;
        for (int half = 0; half < 2; ++half) {
            const int r = half == 0 ? u : p.T - 1 - u;
            if (half == 1 && r == u) break;
            const int row0 = r * 128 + c * 64 + lr0;
            const float nr0 = __ldg(p.norm + row0), nr1 = __ldg(p.norm + row0 + 8);
            double rs[2] = {0.0, 0.0};
            for (int ct = r; ct < p.T; ++ct) {
                float sum[64];
                pair_mma_tile(sum, smem, full, empty, s, ph, c, lane, p.d, ksteps, chunk_len);
                // ---- kernel values, rounded to fp16 once, into R and into this consumer's block (row lr, column j at
                // half j / 64, 16-B chunk ((j % 64) / 8) ^ (lr % 8): the 128-B swizzle)
                const int col0 = ct * 128 + 2 * q;
                float rt[2] = {0.f, 0.f};
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const float2 nc = __ldg(reinterpret_cast<const float2*>(p.norm + col0 + 8 * j));
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        __half kh[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int gi = row0 + 8 * i, gj = col0 + 8 * j + e;
                            const float qd = pair_q(sum[4 * j + 2 * i + e], i ? nr1 : nr0, e ? nc.y : nc.x);
                            float kv;
                            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(kv) : "f"(qd * neg_coef));
                            kh[e] = __float2half_rn(gj > gi && gj < p.N ? kv : 0.f);
                            if constexpr (!kBoot) rt[i] += __half2float(kh[e]);
                        }
                        const int lr = lr0 + 8 * i;
                        const uint32_t addr = kbase + (j >> 3) * (kPermKBytes / 2) + lr * 128 + (((j & 7) ^ (lr & 7)) << 4) + 4 * q;
                        const uint32_t v = (uint32_t)__half_as_ushort(kh[0]) | ((uint32_t)__half_as_ushort(kh[1]) << 16);
                        asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
                    }
                }
                if constexpr (!kBoot) {
                    rs[0] += (double)rt[0];
                    rs[1] += (double)rt[1];
                }
                fence_proxy_async_smem();
                named_bar_sync(2 + c, 128);

                // ---- per block of 64 labellings: U = W_J K^T, then P and C over the rows of I.  bl = labelling row lr0
                // of the block, advanced through an empty asm so that the compiler keeps one pointer live instead of
                // hoisting (and spilling) one per block
                if constexpr (kBoot) {
                    boot_label_product(acc, p, kbase, lr0, q, c, r, ct);
                    named_bar_sync(2 + c, 128);
                    continue;
                }
                const uint32_t* bl = p.bits + (size_t)lr0 * p.words;
                const size_t row8 = 8 * (size_t)p.words, block = (size_t)kPermBlock * p.words;
#pragma unroll
                for (int lb = 0; lb < kPermPass / kPermBlock; ++lb) {
                    if (lb < p.blocks) {
                        const uint4 wj0 = __ldg(reinterpret_cast<const uint4*>(bl + ct * 4));
                        const uint4 wj1 = __ldg(reinterpret_cast<const uint4*>(bl + row8 + ct * 4));
                        const uint32_t j0[4] = {wj0.x, wj0.y, wj0.z, wj0.w}, j1[4] = {wj1.x, wj1.y, wj1.z, wj1.w};
                        // A fragment of k-step kk (columns 16 kk ..): a[0] = labelling row lr0, columns 2 q + {0, 1};
                        // a[1] = row lr0 + 8; a[2], a[3] = columns + 8
                        uint32_t a[8][4];
#pragma unroll
                        for (int kk = 0; kk < 8; ++kk) {
                            const int sh = 16 * (kk & 1) + 2 * q;
                            const uint32_t x0 = j0[kk >> 1] >> sh, x1 = j1[kk >> 1] >> sh;
                            a[kk][0] = perm_half2(x0);
                            a[kk][1] = perm_half2(x1);
                            a[kk][2] = perm_half2(x0 >> 8);
                            a[kk][3] = perm_half2(x1 >> 8);
                        }
                        float dl[32];
                        wgmma_fence();
#pragma unroll
                        for (int kk = 0; kk < 8; ++kk)
                            wgmma_m64n64k16_f16_rs_kmajor(dl, a[kk], kmajor_sw128_desc(kbase + (kk >> 2) * (kPermKBytes / 2)) + 2 * (kk & 3),
                                                          kk > 0);
                        wgmma_commit();
                        wgmma_wait<0>();
                        fence_regs(dl);
                        // element (labelling row lr0 + 8 rr, row 64 c + 8 jj + 2 q + e of I) is dl[4 jj + 2 rr + e]
                        const uint2 wi0 = __ldg(reinterpret_cast<const uint2*>(bl + r * 4 + 2 * c));
                        const uint2 wi1 = __ldg(reinterpret_cast<const uint2*>(bl + row8 + r * 4 + 2 * c));
                        const uint32_t i0[2] = {wi0.x >> (2 * q), wi0.y >> (2 * q)}, i1[2] = {wi1.x >> (2 * q), wi1.y >> (2 * q)};
                        float pp[2] = {0.f, 0.f}, cc[2] = {0.f, 0.f};
#pragma unroll
                        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
                            for (int rr = 0; rr < 2; ++rr) {
                                const uint32_t w = (rr ? i1 : i0)[jj >> 2] >> (8 * (jj & 3));
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const float v = dl[4 * jj + 2 * rr + e];
                                    cc[rr] += v;
                                    pp[rr] += ((w >> e) & 1u) ? v : 0.f;
                                }
                            }
                        }
#pragma unroll
                        for (int o = 1; o < 4; o <<= 1) {
#pragma unroll
                            for (int rr = 0; rr < 2; ++rr) {
                                pp[rr] += __shfl_xor_sync(0xffffffffu, pp[rr], o);
                                cc[rr] += __shfl_xor_sync(0xffffffffu, cc[rr], o);
                            }
                        }
                        // lane q keeps P (q even) or C (q odd) of labelling row lr0 + 8 (q >> 1)
                        const float mine = q == 0 ? pp[0] : q == 1 ? cc[0] : q == 2 ? pp[1] : cc[1];
                        // undo the accumulator's truncation shrink (conv_gemm.cuh): an element of U adds one product
                        // per column the labelling marks (zero products do not truncate); counting every marked
                        // column also counts the masked j <= i ones of a diagonal tile, a shrink of at most
                        // 64 kAccumShrinkPerElement ~ 7e-8 over-corrected there
                        const uint4 jw = q < 2 ? wj0 : wj1;
                        const int marked = __popc(jw.x) + __popc(jw.y) + __popc(jw.z) + __popc(jw.w);
                        acc[lb] += (double)fmaf(mine, kAccumShrinkPerElement * (float)marked, mine);
                        bl += block;
                        asm volatile("" : "+l"(bl));
                    }
                }
                // every warp of this consumer has read the block (wgmma_wait) before the next tile overwrites it
                named_bar_sync(2 + c, 128);
            }
            // R of rows row0, row0 + 8: the quad's 4 lanes by a fixed xor tree
            if constexpr (!kBoot) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    for (int o = 1; o < 4; o <<= 1) rs[i] += __shfl_xor_sync(0xffffffffu, rs[i], o);
                    if (q == 0) p.rowsum[row0 + 8 * i] = rs[i];
                }
            }
        }
        double* part = p.partial + ((size_t)u * 2 + c) * p.blocks * kPermBlock * 2;
#pragma unroll
        for (int lb = 0; lb < kPermPass / kPermBlock; ++lb)
            if (lb < p.blocks) part[(lb * kPermBlock + lr0 + 8 * (q >> 1)) * 2 + (q & 1)] = acc[lb];
    }
}

// one block per labelling (grid = all labellings of the call, padding included); layout and rule above.  Labellings
// b >= 1: an exact radix select (8 passes of 8 bits) of the a-th smallest key K, recomputing the keys each pass; rows
// with key < K are marked, and of the rows with key K the lowest indices until a rows are marked.
__global__ void __launch_bounds__(kPermLabelThreads)
kad_perm_label_kernel(int N, int a, int labellings, unsigned long long seed, int words, uint32_t* __restrict__ bits) {
    __shared__ uint32_t hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ int s_rank;
    __shared__ int s_ties[kPermLabelThreads / 32];
    const int b = blockIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t* out = bits + (size_t)b * words;
    if (b == 0 || b >= labellings) {
        for (int w = threadIdx.x; w < words; w += blockDim.x) {
            const int lo = 32 * w;
            out[w] = b != 0 || lo >= a ? 0u : lo + 32 <= a ? ~0u : (1u << (a - lo)) - 1u;
        }
        return;
    }
    const unsigned long long base = pair_mix64(seed + (unsigned long long)b);
    unsigned long long prefix = 0, mask = 0;
    int rank = a - 1;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int t = threadIdx.x; t < 256; t += blockDim.x) hist[t] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < N; i += blockDim.x) {
            const unsigned long long k = pair_mix64(base ^ (unsigned long long)i);
            if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int below = 0, bin = 0;
            for (; bin < 255; ++bin) {
                if (below + (int)hist[bin] > rank) break;
                below += (int)hist[bin];
            }
            s_prefix = prefix | ((unsigned long long)bin << shift);
            s_rank = rank - below;
        }
        __syncthreads();
        prefix = s_prefix;
        rank = s_rank;
        mask |= 255ull << shift;
    }
    const int take = rank + 1;                      // rows with key == prefix to mark
    int taken = 0;
    for (int i0 = 0; i0 < 32 * words; i0 += blockDim.x) {
        const int i = i0 + threadIdx.x;
        const unsigned long long k = i < N ? pair_mix64(base ^ (unsigned long long)i) : ~0ull;
        const bool tie = i < N && k == prefix;
        const uint32_t tb = __ballot_sync(0xffffffffu, tie);
        if (lane == 0) s_ties[warp] = __popc(tb);
        __syncthreads();
        int before = taken, total = 0;
        for (int w = 0; w < kPermLabelThreads / 32; ++w) {
            if (w < warp) before += s_ties[w];
            total += s_ties[w];
        }
        const bool in = i < N && (k < prefix || (tie && before + __popc(tb & ((1u << lane) - 1u)) < take));
        const uint32_t word = __ballot_sync(0xffffffffu, in);
        if (lane == 0 && (i0 >> 5) + warp < words) out[(i0 >> 5) + warp] = word;
        taken += total;
        __syncthreads();
    }
}

// a fixed-order sum over a block of kPermSumThreads threads (lanes by a shuffle tree, then the warps in order); the
// result in thread 0
__device__ __forceinline__ double perm_block_sum(double s) {
    __shared__ double red[kPermSumThreads / 32];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kPermSumThreads / 32; ++w) t += red[w];
    return t;
}

// one block per labelling: out[b] = the sum of v[i] over the rows labelling b marks; each thread its words in order
// (rows in order within a word), then perm_block_sum
__global__ void __launch_bounds__(kPermSumThreads)
kad_perm_dot_kernel(const uint32_t* __restrict__ bits, int words, const double* __restrict__ v, double* __restrict__ out) {
    const uint32_t* w = bits + (size_t)blockIdx.x * words;
    double s = 0.0;
    for (int k = threadIdx.x; k < words; k += kPermSumThreads) {
        uint32_t x = w[k];
        while (x) {
            s += v[32 * k + __ffs(x) - 1];
            x &= x - 1;
        }
    }
    const double t = perm_block_sum(s);
    if (threadIdx.x == 0) out[blockIdx.x] = t;
}

// *out = sum of v[0 .. n) (one block): each thread its strided values in order, then perm_block_sum
__global__ void __launch_bounds__(kPermSumThreads)
kad_perm_total_kernel(const double* __restrict__ v, int n, double* __restrict__ out) {
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += kPermSumThreads) s += v[i];
    const double t = perm_block_sum(s);
    if (threadIdx.x == 0) *out = t;
}

// this pass's P and C: pc[2 l + k] = the sum over units in order, consumer 0 then 1, of partial[u][c][l][k]
__global__ void kad_perm_reduce_kernel(const double* __restrict__ partial, int units, int n, double* __restrict__ pc) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * n) return;
    double s = 0.0;
    for (int u = 0; u < 2 * units; ++u) s += partial[(size_t)u * 2 * n + t];
    pc[t] = s;
}

// ------------------------------------------------------------------------ bootstrap (DESIGN.md 5.18)
// Resample b of F units: draw t = 0 .. F - 1 picks unit floor(key_b(t) F / 2^64) (the high word of the 128-bit
// product: no modulo bias), key_b(t) = pair_mix64(pair_mix64(seed + b) ^ t); w_b(u) = #{t : the draw picks u}.
// Resample 0 is the observed set, every multiplicity 1.
constexpr int kBootThreads = 256;

// one block per resample b = b0 + blockIdx.x: counts[blockIdx.x][u - u0] = w_b(u) for u in [u0, u0 + width); rows
// b >= resamples (the call's B + 1) are zero.  Integer atomics, so the counts do not depend on the order.  limit > 0:
// *over = 1 when a count exceeds it
__global__ void __launch_bounds__(kBootThreads)
boot_counts_kernel(long long F, long long u0, int width, int b0, int resamples, unsigned long long seed,
                   uint32_t* __restrict__ counts, uint32_t limit, int* __restrict__ over) {
    const int b = b0 + blockIdx.x;
    uint32_t* row = counts + (size_t)blockIdx.x * width;
    for (int k = threadIdx.x; k < width; k += kBootThreads) row[k] = b == 0 ? 1u : 0u;
    if (b == 0 || b >= resamples) return;
    __syncthreads();
    const unsigned long long base = pair_mix64(seed + (unsigned long long)b);
    for (long long t = threadIdx.x; t < F; t += kBootThreads) {
        const long long u = (long long)__umul64hi(pair_mix64(base ^ (unsigned long long)t), (unsigned long long)F) - u0;
        if (u >= 0 && u < width) atomicAdd(row + u, 1u);
    }
    if (limit == 0) return;
    __syncthreads();
    for (int k = threadIdx.x; k < width; k += kBootThreads)
        if (__ldcg(row + k) > limit) *over = 1;
}

// unit_of[i] = the unit of row i (offsets [units + 1]); one thread per unit
__global__ void boot_unit_index_kernel(const long long* __restrict__ offsets, int units, int* __restrict__ unit_of) {
    for (int u = blockIdx.x * blockDim.x + threadIdx.x; u < units; u += gridDim.x * blockDim.x)
        for (long long i = offsets[u]; i < offsets[u + 1]; ++i) unit_of[i] = u;
}

// weights[r][i] = counts[r][unit_of[i]] as fp16 (exact up to 2048), 0 for N <= i < Npad; grid (blocks, rows)
__global__ void boot_weights_kernel(const uint32_t* __restrict__ counts, long long F, const int* __restrict__ unit_of,
                                    int N, int Npad, __half* __restrict__ weights) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= Npad) return;
    const size_t r = blockIdx.y;
    weights[r * Npad + i] = __uint2half_rn(i < N ? counts[r * F + unit_of[i]] : 0u);
}

// one block per resample row of a pass: out[b] = (n_b, Q_b + sum_u n_u w_u (w_u - 1) / 2, sum_u w_u g_u) with
// Q_b = pc[2 b] (the pass's label product), each sum over the units in a fixed order (perm_block_sum)
__global__ void __launch_bounds__(kPermSumThreads)
boot_unit_terms_kernel(const uint32_t* __restrict__ counts, long long F, const long long* __restrict__ offsets,
                       const double* __restrict__ g, const double* __restrict__ pc, double* __restrict__ out) {
    const uint32_t* w = counts + (size_t)blockIdx.x * F;
    double n = 0.0, sxy = 0.0, self = 0.0;
    for (long long u = threadIdx.x; u < F; u += kPermSumThreads) {
        const double wu = (double)w[u], nu = (double)(offsets[u + 1] - offsets[u]);
        n += wu * nu;
        sxy += wu * g[u];
        self += nu * (wu * (wu - 1.0) * 0.5);
    }
    n = perm_block_sum(n);
    __syncthreads();
    sxy = perm_block_sum(sxy);
    __syncthreads();
    self = perm_block_sum(self);
    if (threadIdx.x == 0) {
        double* o = out + 3 * (size_t)blockIdx.x;
        o[0] = n;
        o[1] = pc[2 * (size_t)blockIdx.x] + self;
        o[2] = sxy;
    }
}

// out[b] = (S_aa, S_bb, S_ab) = (P, ((T - L) - C) + P, (L + C) - 2 P) for the first `labellings` labellings
__global__ void kad_perm_finish_kernel(const double* __restrict__ pc, const double* __restrict__ l,
                                       const double* __restrict__ total, int labellings, double* __restrict__ out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= labellings) return;
    const double P = pc[2 * b], C = pc[2 * b + 1], L = l[b], T = *total;
    out[3 * (size_t)b] = P;
    out[3 * (size_t)b + 1] = ((T - L) - C) + P;
    out[3 * (size_t)b + 2] = (L + C) - 2.0 * P;
}

}  // namespace fad
