// Precision, recall, density and coverage (PRDC) of two embedding sets on Hopper tensor cores: the k-nearest-neighbour
// radii of each set and the ball counts between the sets (DESIGN.md section 5.12).
//
// Z = [X; Y] (fp16 [m + n, d], X first).  The distances are the ones KAD computes: the pair-tile prologue (shared fp16
// shift, hi/lo split, fp64 row norms), tile loop (pair_load_tile, pair_mma_tile) and q (pair_q) of pair_tile.cuh.
// Only the epilogue differs, and every output is a selected fp32 value or an integer count, so every pass is bitwise
// reproducible and independent of the grid without any partial-sum bookkeeping.
//
// Radii (PASS 0; per song PASS 2, the same body).  Unit u < Tx: the A operand is X tile u (rows 128 u), the B operands
// are every X tile; unit Tx + t: the A operand is the 128-row tile of Y at row m + 128 t (not tile-aligned in Z), the
// B operands are every Y tile (PASS 2: the song band, 128-row boxes from the first row of the song that owns the
// tile's first row up to the end of the song that owns its last row; song_of[r] = the song of Y row r, -1 past the
// last row).  Each consumer thread holds two rows and keeps, per row, the k smallest q of its columns in a sorted
// register list (an insertion runs only when q is below the current k-th value).  A row counts the columns of its own
// set other than itself (PASS 2: of its own song, the row's range [offsets[s], offsets[s + 1]) of Y, so s_j is the
// radius calc_prdc(X, Y_k) computes for y_j: the same operand orientation and chunking, only the tile position
// differs).  Masks are by index only: the rows the TMA unit zero-fills never count, duplicate rows are neighbours at 0.
// PASS 0 compares no lower bound, at compile time: at d = 128 the epilogue is part of the pass's cost (DESIGN.md 7).
// The full square is run, not the triangle: a column-wise top-k would need a second sorted list per column of the
// fragment, and the unit then owns whole rows.  At the end of the unit the four lanes of a quad (same rows) merge
// their lists by a fixed xor tree, and one lane writes radii_sq[row of Z] = the k-th smallest of the set's q values.
// Selection does not depend on order, so the value is exact and grid-independent.
//
// Radius lists (PASS 6): PASS 0 on X alone (n = 0), but one lane writes the row's whole list, the k smallest q
// ascending, to radii_sq[row][k]: entry k' - 1 is bitwise the PASS 0 radius at k' <= k, both being exact selections
// of the same fp32 values (DESIGN.md 5.15).
//
// Counts (PASS 1).  Unit = (X tile tx, a run of Y column tiles [c0, c1)), runs cut by the shape only.  r_i^2 of the
// two rows of a thread sit in registers; s_j^2 is read per column through the read-only cache, as the column norms
// are.  Every xy pair is evaluated once, so the four metrics see one fp32 q per pair:
//   row i:    covered |= q < r_i^2,   recalled |= q < s_j^2   (ORed over the quad, then atomicOr of 1 into the
//                                                               covered and recalled planes of row_flags at row i)
//   column j: inside[j] += #{i : q < r_i^2}                    (prdc_tally: integer shuffle tree over the 8 row
//                                                               groups of a warp, then integer atomicAdd)
// No floating-point atomic anywhere.  prdc_flags_kernel packs the two planes into the uint8 flags.
//
// Per-song counts (PASS 3).  Unit = (X tile row, span): a span is a run of whole songs cut by the host (spans[]); the B
// boxes start at the span's first row and count the columns of its songs.  inside[j] as in PASS 1.  Per (baseline row,
// song) the covered / recalled decisions are ORed over the song's columns: each thread walks its columns in ascending
// order, so the songs arrive in monotone order; it carries a running (song, flags) pair and, when the song changes,
// atomicOrs nonzero flags into a shared-memory bitmap [songs][128 rows / 32][2 planes].  At the end of the unit the 256
// consumers popcount each song's words into song_counts[song][covered | recalled] (integer atomicAdd) and clear the
// bitmap.  Each (X tile, song) pair belongs to one unit, so no (row, song) pair is counted twice.
//
// Realism (PASS 4, DESIGN.md 5.13).  Unit = (Y tile t, a run of X column tiles [c0, c1)), runs cut by the shape only as
// in PASS 1.  The A operand is the 128-row box of Y at row m + 128 t, so each thread owns two eval rows and reduces
// along the fragment's columns in registers over all the unit's tiles: no per-tile shuffle, no atomic.  Per row it
// keeps the best quotient b = max r~_i^2 / q (r~_i^2, the pruned radius of column i, read through the read-only cache)
// without a division per pair: fmaf(b, q, -r~^2) < 0 is the exact sign of b q - r~^2, and only then is b set to the
// correctly rounded r~^2 / q, so b is exactly the max of fl(r~_i^2 / q) (r~^2 = 0 never improves; q = 0 < r~^2 gives
// +inf; b = +inf, q = 0 gives NaN, which compares false).  And the nearest column (q, i) by a strict < in ascending
// column order.  Columns j >= m (the last X tile runs into Y) count nothing.  At the end of the unit the quad merges
// by a fixed xor tree (max; lexicographic min of (q, i)) and one lane writes the row's slot of this run in part; exactly
// one unit writes each slot.  realism_reduce_kernel takes the max and the lexicographic min over the runs.
//
// Nearest groups (PASS 5, DESIGN.md 5.14).  The units, the orientation and the masks of PASS 4.  The baseline rows are
// cut into groups (contiguous row ranges, song_of = the group of each X row, offsets = the group bounds); per eval row
// the thread keeps the k nearest distinct groups, each by its smallest key (q, row of X), in a sorted list: the q values
// in registers as prdc_insert keeps them (dead entries -inf, empty ones +inf, the k-th at index 15), the rows in the
// kernel's own shared memory (a second list of 16 in registers would spill next to the accumulators).  The common path
// is one compare of q with the k-th q: the thread walks its columns in ascending row order, so a candidate with an equal
// q has the larger key.  The fragment loop only marks such candidates in a mask per row, drained in ascending order at
// one insertion site per row (inlined at every fragment position the kernel ran 11 x slower, out of the instruction
// cache).  Only a candidate that beats the k-th reads its group's bounds (nearest_insert).  At the end of the
// unit the quad merges by a fixed xor tree with the same insertion on full keys, and one lane writes the row's k entries
// of this run in part; exactly one unit writes each slot.  nearest_reduce_kernel merges the runs the same way.  The top
// k groups of a union of column sets are the top k of the merged top-k lists (a group in the union's top k is in the
// top k of the set that attains its minimum), and keys are distinct, so every result is exact and grid-independent.
//
// Shards (pairwise_host.inc, DESIGN.md 5.12).  A launch runs the units [unit0, unit1).  A radii unit owns whole rows, so a
// shard writes exactly its units' radii; a counts shard adds into its own inside and row_flags.  The flags are kept as
// one 0/1 plane per bit, not as packed bits, so that the host can add the shards' copies and read "nonzero" as OR.
//
// Warp roles and stages are the pair-tile ones: warpgroup 0 = TMA producer, warpgroups 1-2 = consumers on rows
// [64 c, 64 c + 64) of the tile.
#pragma once
#include "pair_tile.cuh"

namespace fad {

constexpr int kPrdcMaxK = 16;
static_assert(kPairSmemBytes <= 227 * 1024, "over the per-CTA shared-memory limit");
// PASS 3: at most kPrdcSpanSongs songs per span, a bitmap of [songs][128 / 32 words][2 planes] after the barriers
constexpr int kPrdcSpanSongs = 512;
constexpr uint32_t kPrdcBitmapWords = kPrdcSpanSongs * 4 * 2;
constexpr uint32_t kPrdcSongSmemBytes = kPairSmemBytes + kPrdcBitmapWords * 4;
static_assert(kPrdcSongSmemBytes <= 227 * 1024, "over the per-CTA shared-memory limit");
// PASS 5: the rows of each consumer thread's two lists, [entry][list][consumer thread] words after the barriers
constexpr int kNearestListStride = 2 * 256;
constexpr uint32_t kPrdcNearestSmemBytes = kPairSmemBytes + kPrdcMaxK * kNearestListStride * 4;
static_assert(kPrdcNearestSmemBytes <= 227 * 1024, "over the per-CTA shared-memory limit");

struct PrdcParams {
    int m, n, d;             // rows of X, rows of Y, columns
    int Tx, Ty;              // ceil(m / 128), ceil(n / 128)
    int unit0, unit1;        // this launch's units [unit0, unit1) of Tx + Ty (PASS 0, 2) or Tx * cuts (PASS 1, 3): all
                             // of them, or one shard of a sharded call; outputs stay indexed by the global row / column
    const float* norm;       // [m + Ty * 128] |y_i|^2 of the rows of Z (zero past m + n; per song: one box more)
    // PASS 0, 2 and 6
    int k;                   // 1 .. kPrdcMaxK
    float* radii_sq;         // [m + n] out (PASS 6: [m][k])
    // PASS 1 and 3
    const float* radii;      // [m + n] r_i^2 of X, then s_j^2 of Y
    int cuts;                // column runs per X tile row: run i = Y tiles [i Ty / cuts, (i + 1) Ty / cuts)
    int* inside;             // [n], zeroed by the host
    int* row_flags;          // [2][m], zeroed by the host: plane 0 covered, plane 1 recalled (1 where set)
    // PASS 2 and 3 (per song): n = n_total, the rows of all songs; PASS 3: cuts = the number of spans
    const int* song_of;      // [Ty * 128 + 128] the song of each Y row, -1 past the last row
    const long long* offsets;// [songs + 1] song s = Y rows [offsets[s], offsets[s + 1])
    const int4* spans;       // PASS 3: [cuts] {first Y row, end Y row, first song, songs}
    int* song_counts;        // PASS 3: [songs][2] covered, recalled baseline rows, zeroed by the host
    // PASS 4: radii = [m] the pruned radii r~_i^2 of X; cuts = X column runs per Y tile: run i = X tiles
    // [i Tx / cuts, (i + 1) Tx / cuts)
    uint32_t* part;          // [3][cuts][n] out: per (run, Y row) the bits of the best quotient, of the nearest q, its index
    // PASS 5: cuts as PASS 4; song_of = [Tx * 128] the group of each X row, offsets = [groups + 1] the group bounds in X;
    // part = [2][cuts][n][k] out: per (run, Y row) the k entries' q bits, then their rows (+inf bits, 0xFFFFFFFF: empty)
};

// the tiles of unit u: A rows from arow, B tiles [c0, c1) at rows bbase + 128 c
struct PrdcUnit {
    int arow, bbase, c0, c1;
};
template <int PASS>
__device__ __forceinline__ PrdcUnit prdc_unit(const PrdcParams& p, int u) {
    if constexpr (PASS == 0 || PASS == 6) {
        if (u < p.Tx) return {u * 128, 0, 0, p.Tx};
        return {p.m + (u - p.Tx) * 128, p.m, 0, p.Ty};
    } else if constexpr (PASS == 2) {
        // Y tile t: the band from the first row of the song of row 128 t to the end of the song of its last row
        if (u < p.Tx) return {u * 128, 0, 0, p.Tx};
        const int t = u - p.Tx;
        const int first = (int)__ldg(p.offsets + __ldg(p.song_of + 128 * t));
        const int end = (int)__ldg(p.offsets + __ldg(p.song_of + min(128 * t + 127, p.n - 1)) + 1);
        return {p.m + 128 * t, p.m + first, 0, (end - first + 127) / 128};
    } else if constexpr (PASS == 1) {
        const int tx = u / p.cuts, i = u - tx * p.cuts;
        return {tx * 128, p.m, (int)((long long)i * p.Ty / p.cuts), (int)((long long)(i + 1) * p.Ty / p.cuts)};
    } else if constexpr (PASS == 3) {
        const int tx = u / p.cuts;
        const int4 sp = p.spans[u - tx * p.cuts];
        return {tx * 128, p.m + sp.x, 0, (sp.y - sp.x + 127) / 128};
    } else {
        const int t = u / p.cuts, i = u - t * p.cuts;
        return {p.m + 128 * t, 0, (int)((long long)i * p.Tx / p.cuts), (int)((long long)(i + 1) * p.Tx / p.cuts)};
    }
}

// a[0..15] ascending, the live entries last: q < a[15] replaces the k-th value and moves down to its place (the dead
// entries are -inf and never move, so the list keeps the k smallest values in a[16 - k .. 15])
__device__ __forceinline__ void prdc_insert(float (&a)[kPrdcMaxK], float q) {
    a[kPrdcMaxK - 1] = q;
#pragma unroll
    for (int s = kPrdcMaxK - 1; s > 0; --s) {
        const float lo = fminf(a[s - 1], a[s]), hi = fmaxf(a[s - 1], a[s]);
        a[s - 1] = lo;
        a[s] = hi;
    }
}

// the 4 lanes of a quad hold the same two rows over disjoint columns: merge by a fixed xor tree (each lane takes a
// snapshot of its partner's list first, then inserts its live entries)
__device__ __forceinline__ void prdc_topk_merge(float (&a)[2][kPrdcMaxK]) {
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float b[kPrdcMaxK];
#pragma unroll
            for (int t = 0; t < kPrdcMaxK; ++t) b[t] = __shfl_xor_sync(0xffffffffu, a[i][t], o);
#pragma unroll
            for (int t = 0; t < kPrdcMaxK; ++t)
                if (b[t] >= 0.f && b[t] < a[i][kPrdcMaxK - 1]) prdc_insert(a[i], b[t]);
        }
    }
}

// nearest groups: the rows of a list, in the kernel's shared memory (stride kNearestListStride) or in registers; the
// index is always a compile-time constant
struct NearestSmemRows {
    uint32_t* p;
    __device__ __forceinline__ uint32_t get(int t) const { return p[t * kNearestListStride]; }
    __device__ __forceinline__ void set(int t, uint32_t v) const { p[t * kNearestListStride] = v; }
};
struct NearestRegRows {
    uint32_t (&r)[kPrdcMaxK];
    __device__ __forceinline__ uint32_t get(int t) const { return r[t]; }
    __device__ __forceinline__ void set(int t, uint32_t v) const { r[t] = v; }
};

// key (q, row) below key (qb, rb): the fp32 order of q >= 0, then the row
__device__ __forceinline__ bool nearest_less(float q, uint32_t row, float qb, uint32_t rb) {
    return q < qb || (q == qb && row < rb);
}

// a[0..15] / r ascending by key, the live entries last as in prdc_insert (dead: -inf, empty: +inf, both row 0xFFFFFFFF,
// which lies in no group), at most one entry per group.  The candidate (q, row), row < m, has a key below the k-th
// (a[15], r[15]).  If its group has an entry, the candidate replaces it when its key is smaller and is dropped
// otherwise; else it replaces the k-th entry.  One compare-exchange sweep then moves it to its place.
template <typename Rows>
__device__ __forceinline__ void nearest_insert(float (&a)[kPrdcMaxK], const Rows& r, float q, uint32_t row,
                                               const int* __restrict__ song_of, const long long* __restrict__ offsets) {
    const int g = __ldg(song_of + row);
    const uint32_t lo = (uint32_t)__ldg(offsets + g), span = (uint32_t)__ldg(offsets + g + 1) - lo;
    int at = kPrdcMaxK - 1;
    bool drop = false;
#pragma unroll
    for (int t = 0; t < kPrdcMaxK; ++t) {
        const uint32_t rt = r.get(t);
        if (rt - lo < span) {
            if (nearest_less(a[t], rt, q, row)) drop = true;
            else at = t;
        }
    }
    if (drop) return;
#pragma unroll
    for (int t = 0; t < kPrdcMaxK; ++t)
        if (t == at) { a[t] = q; r.set(t, row); }
#pragma unroll
    for (int s = kPrdcMaxK - 1; s > 0; --s) {
        if (s <= at && (a[s - 1] > a[s] || (a[s - 1] == a[s] && r.get(s - 1) > r.get(s)))) {
            const float t = a[s - 1];
            a[s - 1] = a[s];
            a[s] = t;
            const uint32_t lo_row = r.get(s), hi_row = r.get(s - 1);
            r.set(s - 1, lo_row);
            r.set(s, hi_row);
        }
    }
}

// counts: the decisions of one xy pair from its dot product and norms, bit 0 q < r2 (where the column counts), bit 1
// q < s2 (where the row counts).  r2 = 0 for a row past m and s2 = 0 for a column that does not count: q < 0 is never
// true
__device__ __forceinline__ uint32_t prdc_pair(float dot, float nr, float nc, float r2, float s2, bool col_ok, bool row_ok) {
    const float q = pair_q(dot, nr, nc);
    return (uint32_t)(q < r2 && col_ok) | ((uint32_t)(row_ok && q < s2) << 1);
}

// counts: inside[jj] += the low 16 bits of cj, inside[jj + 1] += the high 16 bits, summed over the warp.  Rarely taken:
// the 8 row groups of the warp hold the same columns, lanes l, l ^ 4, ..., l ^ 28 (at most 16 rows per column, so the
// two 16-bit halves do not carry into each other)
__device__ __forceinline__ void prdc_tally(uint32_t cj, int* inside, int jj, int lane) {
    if (__any_sync(0xffffffffu, cj != 0)) {
        for (int o = 4; o < 32; o <<= 1) cj += __shfl_xor_sync(0xffffffffu, cj, o);
        if (lane < 4) {
            if (cj & 0xFFFFu) atomicAdd(inside + jj, (int)(cj & 0xFFFFu));
            if (cj >> 16) atomicAdd(inside + jj + 1, (int)(cj >> 16));
        }
    }
}

template <int PASS>
__global__ void __launch_bounds__(kPairThreads, 1)
prdc_tile_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo, const PrdcParams p) {
    using namespace sm90;
    static_assert(PASS >= 0 && PASS <= 6, "0: k-NN radii, 1: ball counts, 2: per-song radii, 3: per-song counts, "
                  "4: realism, 5: nearest groups, 6: k-NN radius lists");
    extern __shared__ uint8_t smem_raw[];
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const PairTile pt = pair_tile_open(smem_raw, &map_hi, &map_lo, p.d, warp, lane);
    uint8_t* smem = pt.smem;
    uint64_t* full = pt.full;
    uint64_t* empty = pt.empty;
    const int ksteps = pt.ksteps, chunk_len = pt.chunk_len;
    uint32_t* bitmap = reinterpret_cast<uint32_t*>(pt.own);        // PASS 3
    if constexpr (PASS == 3)
        for (int b = threadIdx.x; b < (int)kPrdcBitmapWords; b += kPairThreads) bitmap[b] = 0;
    __syncthreads();

    if (warp < 4) {
        // ------------------------------------------------------------ TMA producer
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            int s = 0; uint32_t ph = 0;
            for (int u = p.unit0 + blockIdx.x; u < p.unit1; u += gridDim.x) {
                const PrdcUnit w = prdc_unit<PASS>(p, u);
                for (int ct = w.c0; ct < w.c1; ++ct)
                    pair_load_tile(smem, full, empty, s, ph, &map_hi, &map_lo, ksteps, w.arow, w.bbase + ct * 128);
            }
        }
        return;
    }
    // ---------------------------------------------------------------- consumers: wgmma + epilogue in registers
    setmaxnreg_inc<kPairConsumerRegs>();
    const int c = (warp >> 2) - 1;                        // tile rows [64 c, 64 c + 64)
    const int lr0 = c * 64 + (warp & 3) * 16 + (lane >> 2);   // tile rows lr0, lr0 + 8
    int s = 0; uint32_t ph = 0;
    for (int u = p.unit0 + blockIdx.x; u < p.unit1; u += gridDim.x) {
        const PrdcUnit w = prdc_unit<PASS>(p, u);
        const int row0 = w.arow + lr0;                    // rows of Z
        const float nr[2] = {__ldg(p.norm + row0), __ldg(p.norm + row0 + 8)};
        if constexpr (PASS == 0 || PASS == 2 || PASS == 6) {
            // each row's set as a range [lo, hi) of the unit's columns jj (rows bbase + jj of Z): the whole set (lo = 0
            // is not compared); per song, for the Y units, the row's song, empty past the last row (song_of = -1)
            constexpr bool songs = PASS == 2;
            const int ii0 = row0 - w.bbase;               // the rows' own columns
            int lo[2], hi[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                if (!songs || w.bbase == 0) {
                    lo[i] = 0;
                    hi[i] = w.bbase == 0 ? p.m : p.n;
                } else {
                    const int sg = __ldg(p.song_of + row0 + 8 * i - p.m);
                    lo[i] = sg < 0 ? 0 : p.m + (int)__ldg(p.offsets + sg) - w.bbase;
                    hi[i] = sg < 0 ? 0 : p.m + (int)__ldg(p.offsets + sg + 1) - w.bbase;
                }
            }
            float a[2][kPrdcMaxK];
#pragma unroll
            for (int t = 0; t < kPrdcMaxK; ++t) {
                a[0][t] = a[1][t] = t < kPrdcMaxK - p.k ? -INFINITY : INFINITY;
            }
            for (int ct = w.c0; ct < w.c1; ++ct) {
                float sum[64];
                pair_mma_tile(sum, smem, full, empty, s, ph, c, lane, p.d, ksteps, chunk_len);
                // element (row0 + 8 i, column jj0 + 8 j + e) is sum[4 j + 2 i + e]
                const int jj0 = ct * 128 + 2 * (lane & 3);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    // the Y part starts at row m, of any parity: two scalar loads, not a float2
                    const float nc[2] = {__ldg(p.norm + w.bbase + jj0 + 8 * j), __ldg(p.norm + w.bbase + jj0 + 8 * j + 1)};
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int jj = jj0 + 8 * j + e;
                            const float q = pair_q(sum[4 * j + 2 * i + e], nr[i], nc[e]);
                            if ((!songs || jj >= lo[i]) && jj < hi[i] && jj != ii0 + 8 * i && q < a[i][kPrdcMaxK - 1])
                                prdc_insert(a[i], q);
                        }
                    }
                }
            }
            prdc_topk_merge(a);
            if ((lane & 3) == 0) {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    if ((!songs || ii0 + 8 * i >= lo[i]) && ii0 + 8 * i < hi[i]) {
                        if constexpr (PASS == 6) {
#pragma unroll
                            for (int t = 0; t < kPrdcMaxK; ++t)
                                if (t >= kPrdcMaxK - p.k)
                                    p.radii_sq[(size_t)(row0 + 8 * i) * p.k + t - (kPrdcMaxK - p.k)] = a[i][t];
                        } else {
                            p.radii_sq[row0 + 8 * i] = a[i][kPrdcMaxK - 1];
                        }
                    }
                }
            }
        } else if constexpr (PASS == 1) {
            // rows of X past m (the first rows of Y, or zero-filled) count nothing
            const bool rv[2] = {row0 < p.m, row0 + 8 < p.m};
            const float r2[2] = {rv[0] ? __ldg(p.radii + row0) : 0.f, rv[1] ? __ldg(p.radii + row0 + 8) : 0.f};
            bool cov[2] = {false, false}, rec[2] = {false, false};
            for (int ct = w.c0; ct < w.c1; ++ct) {
                float sum[64];
                pair_mma_tile(sum, smem, full, empty, s, ph, c, lane, p.d, ksteps, chunk_len);
                const int jj0 = ct * 128 + 2 * (lane & 3);    // rows of Y
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int jj = jj0 + 8 * j;
                    const float nc[2] = {__ldg(p.norm + p.m + jj), __ldg(p.norm + p.m + jj + 1)};
                    const float s2[2] = {jj < p.n ? __ldg(p.radii + p.m + jj) : 0.f,
                                         jj + 1 < p.n ? __ldg(p.radii + p.m + jj + 1) : 0.f};
                    uint32_t cj = 0;                          // column jj in bits 0-15, jj + 1 in bits 16-31
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const uint32_t b = prdc_pair(sum[4 * j + 2 * i + e], nr[i], nc[e], r2[i], s2[e], jj + e < p.n, rv[i]);
                            cov[i] |= b & 1u;
                            rec[i] |= b >> 1;
                            cj += (b & 1u) << (16 * e);
                        }
                    }
                    prdc_tally(cj, p.inside, jj, lane);
                }
            }
            uint32_t bits[2] = {(uint32_t)cov[0] | ((uint32_t)rec[0] << 1), (uint32_t)cov[1] | ((uint32_t)rec[1] << 1)};
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                for (int o = 1; o < 4; o <<= 1) bits[i] |= __shfl_xor_sync(0xffffffffu, bits[i], o);
                if ((lane & 3) == 0) {
                    if (bits[i] & 1u) atomicOr(p.row_flags + row0 + 8 * i, 1);
                    if (bits[i] & 2u) atomicOr(p.row_flags + p.m + row0 + 8 * i, 1);
                }
            }
        } else if constexpr (PASS == 4) {
            float best[2] = {0.f, 0.f};                       // max r~^2 / q so far
            float nq[2] = {INFINITY, INFINITY};               // the nearest column's q and index
            int ni[2] = {INT_MAX, INT_MAX};
            for (int ct = w.c0; ct < w.c1; ++ct) {
                float sum[64];
                pair_mma_tile(sum, smem, full, empty, s, ph, c, lane, p.d, ksteps, chunk_len);
                const int jj0 = ct * 128 + 2 * (lane & 3);    // rows of X
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int jj = jj0 + 8 * j;
                    const float nc[2] = {__ldg(p.norm + jj), __ldg(p.norm + jj + 1)};
                    const float r2[2] = {jj < p.m ? __ldg(p.radii + jj) : 0.f, jj + 1 < p.m ? __ldg(p.radii + jj + 1) : 0.f};
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const float q = pair_q(sum[4 * j + 2 * i + e], nr[i], nc[e]);
                            if (fmaf(best[i], q, -r2[e]) < 0.f) best[i] = r2[e] / q;
                            if (q < nq[i] && jj + e < p.m) { nq[i] = q; ni[i] = jj + e; }
                        }
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                for (int o = 1; o < 4; o <<= 1) {
                    const float b = __shfl_xor_sync(0xffffffffu, best[i], o);
                    const float oq = __shfl_xor_sync(0xffffffffu, nq[i], o);
                    const int oi = __shfl_xor_sync(0xffffffffu, ni[i], o);
                    best[i] = fmaxf(best[i], b);
                    if (oq < nq[i] || (oq == nq[i] && oi < ni[i])) { nq[i] = oq; ni[i] = oi; }
                }
                const int r = row0 + 8 * i - p.m;             // row of Y
                if ((lane & 3) == 0 && r < p.n) {
                    const size_t slot = (size_t)(u % p.cuts) * p.n + r, plane = (size_t)p.cuts * p.n;
                    p.part[slot] = __float_as_uint(best[i]);
                    p.part[plane + slot] = __float_as_uint(nq[i]);
                    p.part[2 * plane + slot] = (uint32_t)ni[i];
                }
            }
        } else if constexpr (PASS == 5) {
            // list i: q values in a[i], rows in shared memory at [t][i][consumer thread]
            const NearestSmemRows rows[2] = {{reinterpret_cast<uint32_t*>(pt.own) + (threadIdx.x - 128)},
                                             {reinterpret_cast<uint32_t*>(pt.own) + 256 + (threadIdx.x - 128)}};
            float a[2][kPrdcMaxK];
#pragma unroll
            for (int t = 0; t < kPrdcMaxK; ++t) {
                a[0][t] = a[1][t] = t < kPrdcMaxK - p.k ? -INFINITY : INFINITY;
                rows[0].set(t, 0xFFFFFFFFu);
                rows[1].set(t, 0xFFFFFFFFu);
            }
            for (int ct = w.c0; ct < w.c1; ++ct) {
                float sum[64];
                pair_mma_tile(sum, smem, full, empty, s, ph, c, lane, p.d, ksteps, chunk_len);
                const int jj0 = ct * 128 + 2 * (lane & 3);    // rows of X: column 2 j + e of the thread is row jj0 + 8 j + e
                // q in place of the dot products; hit[i] bit 2 j + e: the pair beats row i's k-th q
                uint32_t hit[2] = {0u, 0u};
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int jj = jj0 + 8 * j;
                    const float nc[2] = {__ldg(p.norm + jj), __ldg(p.norm + jj + 1)};
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const float q = pair_q(sum[4 * j + 2 * i + e], nr[i], nc[e]);
                            sum[4 * j + 2 * i + e] = q;
                            if (q < a[i][kPrdcMaxK - 1] && jj + e < p.m) hit[i] |= 1u << (2 * j + e);
                        }
                    }
                }
                // the candidates in ascending row order, each against the k-th as it is then: one insertion site per
                // row, so the unrolled loop above stays small
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    while (hit[i]) {
                        const int b = __ffs(hit[i]) - 1;
                        hit[i] &= hit[i] - 1;
                        float q = 0.f;
#pragma unroll
                        for (int t = 0; t < 32; ++t)
                            if (t == b) q = sum[4 * (t >> 1) + 2 * i + (t & 1)];
                        if (q < a[i][kPrdcMaxK - 1])
                            nearest_insert(a[i], rows[i], q, (uint32_t)(jj0 + 8 * (b >> 1) + (b & 1)), p.song_of, p.offsets);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                for (int o = 1; o < 4; o <<= 1) {
                    float bq[kPrdcMaxK];
                    uint32_t br[kPrdcMaxK];
#pragma unroll
                    for (int t = 0; t < kPrdcMaxK; ++t) {
                        bq[t] = __shfl_xor_sync(0xffffffffu, a[i][t], o);
                        br[t] = __shfl_xor_sync(0xffffffffu, rows[i].get(t), o);
                    }
                    // the partner's live entries, ascending: the first that does not beat the k-th ends the merge
                    for (int t = kPrdcMaxK - p.k; t < kPrdcMaxK; ++t) {
                        float q = 0.f;
                        uint32_t row = 0u;
#pragma unroll
                        for (int v = 0; v < kPrdcMaxK; ++v)
                            if (v == t) { q = bq[v]; row = br[v]; }
                        if (!nearest_less(q, row, a[i][kPrdcMaxK - 1], rows[i].get(kPrdcMaxK - 1))) break;
                        nearest_insert(a[i], rows[i], q, row, p.song_of, p.offsets);
                    }
                }
                const int r = row0 + 8 * i - p.m;             // row of Y
                if ((lane & 3) == 0 && r < p.n) {
                    const size_t slot = ((size_t)(u % p.cuts) * p.n + r) * p.k, plane = (size_t)p.cuts * p.n * p.k;
#pragma unroll
                    for (int t = 0; t < kPrdcMaxK; ++t) {
                        if (t >= kPrdcMaxK - p.k) {
                            p.part[slot + t - (kPrdcMaxK - p.k)] = __float_as_uint(a[i][t]);
                            p.part[plane + slot + t - (kPrdcMaxK - p.k)] = rows[i].get(t);
                        }
                    }
                }
            }
        } else {
            const int4 sp = p.spans[u % p.cuts];             // Y rows [sp.x, sp.y), songs [sp.z, sp.z + sp.w)
            const bool rv[2] = {row0 < p.m, row0 + 8 < p.m};
            const float r2[2] = {rv[0] ? __ldg(p.radii + row0) : 0.f, rv[1] ? __ldg(p.radii + row0 + 8) : 0.f};
            // the running (song, flags) pair; flags per row: bit 0 covered, bit 1 recalled
            int cur = -1;
            uint32_t fl[2] = {0u, 0u};
            const auto flush = [&]() {
                if (cur >= 0 && (fl[0] | fl[1])) {
                    uint32_t* b = bitmap + (cur - sp.z) * 8;
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int lr = lr0 + 8 * i;
                        if (fl[i] & 1u) atomicOr(b + (lr >> 5) * 2, 1u << (lr & 31));
                        if (fl[i] & 2u) atomicOr(b + (lr >> 5) * 2 + 1, 1u << (lr & 31));
                    }
                }
            };
            for (int ct = w.c0; ct < w.c1; ++ct) {
                float sum[64];
                pair_mma_tile(sum, smem, full, empty, s, ph, c, lane, p.d, ksteps, chunk_len);
                const int jj0 = sp.x + ct * 128 + 2 * (lane & 3);   // rows of Y
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int jj = jj0 + 8 * j;
                    const float nc[2] = {__ldg(p.norm + p.m + jj), __ldg(p.norm + p.m + jj + 1)};
                    // the columns of the span's songs count (song_of = -1 past the last row)
                    const int sg[2] = {__ldg(p.song_of + jj), __ldg(p.song_of + jj + 1)};
                    const bool ok[2] = {sg[0] >= sp.z && sg[0] < sp.z + sp.w, sg[1] >= sp.z && sg[1] < sp.z + sp.w};
                    const float s2[2] = {ok[0] ? __ldg(p.radii + p.m + jj) : 0.f, ok[1] ? __ldg(p.radii + p.m + jj + 1) : 0.f};
                    uint32_t cj = 0;                          // as in PASS 1
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        uint32_t b[2];
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            b[i] = prdc_pair(sum[4 * j + 2 * i + e], nr[i], nc[e], r2[i], s2[e], ok[e], rv[i]);
                            cj += (b[i] & 1u) << (16 * e);
                        }
                        if (ok[e]) {
                            if (sg[e] != cur) {
                                flush();
                                cur = sg[e];
                                fl[0] = fl[1] = 0u;
                            }
                            fl[0] |= b[0];
                            fl[1] |= b[1];
                        }
                    }
                    prdc_tally(cj, p.inside, jj, lane);
                }
            }
            flush();
            // every consumer's flags are in the bitmap: count each (song, plane), then clear it for the next unit
            const int ct_id = threadIdx.x - 128;
            named_bar_sync(1, 256);
            for (int e = ct_id; e < 2 * sp.w; e += 256) {
                uint32_t* b = bitmap + (e >> 1) * 8 + (e & 1);
                const int cnt = __popc(b[0]) + __popc(b[2]) + __popc(b[4]) + __popc(b[6]);
                b[0] = b[2] = b[4] = b[6] = 0u;
                if (cnt) atomicAdd(p.song_counts + 2 * (sp.z + (e >> 1)) + (e & 1), cnt);
            }
            named_bar_sync(1, 256);
        }
    }
}

// flags[i] = bit 0 covered, bit 1 recalled: a plane entry is the number of shards that set it (1 unsharded), so a
// nonzero entry is the OR over the shards
__global__ void prdc_flags_kernel(const int* __restrict__ row_flags, int m, unsigned char* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) flags[i] = (unsigned char)((row_flags[i] != 0) | ((row_flags[m + i] != 0) << 1));
}

// realism: r~_i^2 = r_i^2 where r_i^2 <= t (the median, fp64), 0 otherwise, in place
__global__ void realism_prune_kernel(float* __restrict__ radii_sq, int m, double t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m && !((double)radii_sq[i] <= t)) radii_sq[i] = 0.f;
}

// realism: per Y row the max of the runs' quotients and the lexicographic min of their (nearest q bits, index); both
// exact, so the outputs do not depend on the cut or the grid
__global__ void realism_reduce_kernel(const uint32_t* __restrict__ part, int cuts, int n, float* __restrict__ realism,
                                      int* __restrict__ nearest, float* __restrict__ nearest_sq) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const size_t plane = (size_t)cuts * n;
    float b = 0.f;
    unsigned long long key = ~0ull;
    for (int i = 0; i < cuts; ++i) {
        const size_t s = (size_t)i * n + r;
        b = fmaxf(b, __uint_as_float(part[s]));
        key = min(key, ((unsigned long long)part[plane + s] << 32) | part[2 * plane + s]);
    }
    realism[r] = sqrtf(b);
    nearest[r] = (int)(uint32_t)key;
    nearest_sq[r] = __uint_as_float((uint32_t)(key >> 32));
}

// nearest groups: per Y row the runs' lists (part as PASS 5 writes it) merged by nearest_insert in run order, each
// list's entries ascending, so the first that does not beat the k-th ends it; nearest [n][k] = the rows (-1: empty),
// nearest_sq [n][k] = their q (+inf: empty)
__global__ void nearest_reduce_kernel(const uint32_t* __restrict__ part, int cuts, int n, int k,
                                      const int* __restrict__ song_of, const long long* __restrict__ offsets,
                                      int* __restrict__ nearest, float* __restrict__ nearest_sq) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    float a[kPrdcMaxK];
    uint32_t rows[kPrdcMaxK];
#pragma unroll
    for (int t = 0; t < kPrdcMaxK; ++t) {
        a[t] = t < kPrdcMaxK - k ? -INFINITY : INFINITY;
        rows[t] = 0xFFFFFFFFu;
    }
    const NearestRegRows list{rows};
    const size_t plane = (size_t)cuts * n * k;
    for (int i = 0; i < cuts; ++i) {
        const size_t s = ((size_t)i * n + r) * k;
        for (int t = 0; t < k; ++t) {
            const float q = __uint_as_float(part[s + t]);
            const uint32_t row = part[plane + s + t];
            if (!nearest_less(q, row, a[kPrdcMaxK - 1], rows[kPrdcMaxK - 1])) break;
            nearest_insert(a, list, q, row, song_of, offsets);
        }
    }
#pragma unroll
    for (int t = 0; t < kPrdcMaxK; ++t) {
        if (t >= kPrdcMaxK - k) {
            nearest[(size_t)r * k + t - (kPrdcMaxK - k)] = (int)rows[t];
            nearest_sq[(size_t)r * k + t - (kPrdcMaxK - k)] = a[t];
        }
    }
}

}  // namespace fad
