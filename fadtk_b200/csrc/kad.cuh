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

}  // namespace fad
