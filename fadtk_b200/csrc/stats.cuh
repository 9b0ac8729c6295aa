// Sufficient statistics of an embedding matrix E[N, d] (fp16):   n,  sum(x - s),  sum(y y^T)   with y = x - s and
// s a shared fp16 shift vector.  Replaces np.mean / np.cov in fadtk/fad.py:42-48 and the per-file scatter + Chan
// merge in fadtk/utils.py:13-46 with one shifted E^T E contraction.
//
// Two kernels compute the same packed accumulator (fad_stats_accumulate's `tensor_core`):
//
// stats_dmma_kernel<In>  (0, the product path)   fp64 tensor pipe.  x and s are fp16, so y = x - s is exact
//   in fp64; products and sums are fp64 (mma.sync m8n8k4.f64 -> SASS DMMA.8x8x4): the result is the Gram matrix of
//   the data to ~1e-16, hence positive semi-definite.  Parity needs that: a covariance with cond ~1e9 (CLAP/MERT) or
//   a rank-deficient per-song covariance perturbed at the 1e-6 level of an fp32-accumulating path is indefinite -
//   Newton-Schulz diverges on it and tr sqrt(C1 C2) moves by percents.  One CTA = (64x64 output tile ti <= tj, row
//   range); Y tiles are staged in shared memory as doubles with pitch 68 (== 4 mod 16: conflict-free fragment loads)
//   and double-buffered; each job's tile goes to a workspace and stats_dmma_reduce_kernel sums the jobs in a fixed
//   order (deterministic).  In = double with no shift is the variant score() feeds with per-file fp16-rounded means
//   (fad_stats_accumulate_f64).
//
// stats_simt_kernel  (2)   fp64 CUDA-core contraction of the exact y, with atomics: the independent cross-check of
//   the DMMA kernel (tests/test_gpu_kernels.py compares the two).
//
// song_stats_dmma_kernel runs the same DMMA Gram tile (gram_tile) per song for fad_frechet_batched and finishes each
// song's mean and covariance in place; song_stats_kernel is its CUDA-core form for d not a multiple of 64.
//
// Packed accumulator (fp64, the caller's, all-reduced across GPUs as-is):
//   acc[0] = n,  acc[1 .. d] = sum(x - s) (exact),  acc[1+d .. 1+d+d*d) = sum(y y^T)
//   (d x d, full, row-major),  acc[1+d+d*d ..] = sum y  (centring term of the covariance; the same values as
//   acc[1 .. d], kept so that the layout and the all-reduce length stay as they are)
#pragma once
#include "sm90.cuh"

namespace fad {

__device__ __forceinline__ void pair_to_tiles(int pair, int n_tiles, int& ti, int& tj) {
    ti = 0;
    int rem = pair;
    while (rem >= n_tiles - ti) { rem -= n_tiles - ti; ++ti; }
    tj = ti + rem;
}

// --------------------------------------------------------------------------------------
// gram_tile / stats_dmma_kernel: the product default.  EXACT Gram matrix on the FP64 tensor pipe.
//   y = x - s is exact in fp64 for any two fp16 values (<= 22 significant bits), every product
//   y_a y_b is exact (<= 44 bits), and mma.sync m8n8k4 f64 (SASS DMMA.8x8x4) accumulates in fp64 in
//   a fixed order: the result is the Gram matrix of the data to ~1e-16 - positive semi-definite, which
//   is what Newton-Schulz on cond-1e9 / rank-deficient covariances needs (see the header) - at the
//   tensor-pipe rate instead of the CUDA-core DFMA rate, with no atomics (bit-reproducible).
// One CTA = one job = (64 x 64 output tile (ti <= tj), row range).  256 threads = 8 warps as 2 x 4,
// a warp owns 32 x 16 outputs (4 x 2 DMMA blocks).  E is row-major [row][col]: for E^T E both operand
// fragments read smem as Y[k = row][m or n = col] with pitch 68 doubles (= 4 mod 16: the m8n8k4
// fragment pattern k = lane%4, m = lane/4 touches 16 distinct 8-byte banks per half-warp).
// Loads: 8 bytes (4 fp16) per thread and panel, coalesced 128-B row segments, converted and shifted on
// the way into shared memory; the next 16-row stage is in flight while the current one is multiplied.
// Column sums of y come from the loader's own registers (no extra smem reads).
// Jobs write their fp64 tile to a workspace; stats_dmma_reduce_kernel sums row splits in a fixed order.
constexpr int kSdTile = 64, kSdRows = 16, kSdPitch = kSdTile + 4;

struct StatsDmmaParams {
    long long n_rows;
    int d, n_tiles, n_pairs, n_splits;
    long long rows_per_split;      // multiple of kSdRows
    const __half* shift;           // [d]
    double* ws_tiles;              // [n_pairs * n_splits][64 (row of the tile)][64 (col)]
    double* ws_sums;               // [n_tiles * n_splits][64]
};

typedef double GramStage[2][2][kSdRows][kSdPitch];              // [panel i | j][buffer][row][col]

// The Gram tile both DMMA statistics kernels run: c += Y_i^T Y_j over rows [row_begin, row_end) of E (row pitch d),
// Y_i / Y_j = columns [64 ti, 64 ti + 64) / [64 tj, 64 tj + 64) minus the shift row (none if shift is null).
// In = __half (embeddings) or double (per-file mean rows, no shift).  On return c holds this thread's DMMA
// accumulator fragments and cs_i / cs_j its loader partial column sums of Y_i / Y_j (cs_j = cs_i on the diagonal);
// the stage buffers are free.  Called by all 256 threads.
template <typename In>
__device__ __forceinline__ void gram_tile(GramStage& Ys, const In* __restrict__ E, int d, long long row_begin,
                                          long long row_end, int ti, int tj, const __half* __restrict__ shift,
                                          double (&c)[4][2][2], double (&cs_i)[4], double (&cs_j)[4])
{
    constexpr bool kHalf = sizeof(In) == 2;
    const bool diag = ti == tj;
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
    const int fr = lane >> 2, fk = lane & 3;
    const int lrow = t >> 4, lcol = (t & 15) * 4;               // loader: row of the stage, first of 4 columns

    double si[4] = {0.0, 0.0, 0.0, 0.0}, sj[4] = {0.0, 0.0, 0.0, 0.0};
    if (kHalf && shift != nullptr) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            si[e] = (double)__half2float(shift[ti * kSdTile + lcol + e]);
            sj[e] = (double)__half2float(shift[tj * kSdTile + lcol + e]);
        }
    }
    const In* src_i = E + (size_t)ti * kSdTile + lcol;
    const In* src_j = E + (size_t)tj * kSdTile + lcol;
    double ri[4] = {0.0, 0.0, 0.0, 0.0}, rj[4] = {0.0, 0.0, 0.0, 0.0};        // the 4 values of this thread, already as fp64
    bool rok = false;
    auto load4 = [&](const In* ptr, double (&v)[4]) {
        if constexpr (kHalf) {
            const uint2 raw = __ldg(reinterpret_cast<const uint2*>(ptr));
            const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
            const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
            v[0] = (double)f0.x; v[1] = (double)f0.y; v[2] = (double)f1.x; v[3] = (double)f1.y;
        } else {
            const double2 a = __ldg(reinterpret_cast<const double2*>(ptr)), b = __ldg(reinterpret_cast<const double2*>(ptr) + 1);
            v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
        }
    };
    auto fetch = [&](long long r0) {
        const long long r = r0 + lrow;
        rok = r < row_end;
        if (rok) {
            load4(src_i + (size_t)r * d, ri);
            if (!diag) load4(src_j + (size_t)r * d, rj);
        }
    };
    auto stage = [&](int buf) {
        double y[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) y[e] = rok ? ri[e] - si[e] : 0.0;
        *reinterpret_cast<double2*>(&Ys[0][buf][lrow][lcol]) = make_double2(y[0], y[1]);
        *reinterpret_cast<double2*>(&Ys[0][buf][lrow][lcol + 2]) = make_double2(y[2], y[3]);
#pragma unroll
        for (int e = 0; e < 4; ++e) cs_i[e] += y[e];
        if (!diag) {
#pragma unroll
            for (int e = 0; e < 4; ++e) y[e] = rok ? rj[e] - sj[e] : 0.0;
            *reinterpret_cast<double2*>(&Ys[1][buf][lrow][lcol]) = make_double2(y[0], y[1]);
            *reinterpret_cast<double2*>(&Ys[1][buf][lrow][lcol + 2]) = make_double2(y[2], y[3]);
#pragma unroll
            for (int e = 0; e < 4; ++e) cs_j[e] += y[e];
        }
    };

    const int stages = row_end > row_begin ? (int)((row_end - row_begin + kSdRows - 1) / kSdRows) : 0;
    if (stages > 0) {
        fetch(row_begin);
        stage(0);
    }
    __syncthreads();
    const int bp = diag ? 0 : 1;
    for (int st = 0; st < stages; ++st) {
        const int buf = st & 1;
        if (st + 1 < stages) fetch(row_begin + (long long)(st + 1) * kSdRows);
#pragma unroll
        for (int kk = 0; kk < kSdRows; kk += 4) {
            double a[4], b[2];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = Ys[0][buf][kk + fk][wm + i * 8 + fr];
#pragma unroll
            for (int j = 0; j < 2; ++j) b[j] = Ys[bp][buf][kk + fk][wn + j * 8 + fr];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j) sm90::dmma_884(c[i][j][0], c[i][j][1], a[i], b[j]);
        }
        if (st + 1 < stages) stage(buf ^ 1);
        __syncthreads();
    }
    if (diag) {
#pragma unroll
        for (int e = 0; e < 4; ++e) cs_j[e] = cs_i[e];
    }
}

// Column sums of Y over the tile's rows: the 16 loader partials of each column added in a fixed order, through the
// stage buffers gram_tile left free.  Thread t < 64 panels returns the sum of column t % 64 of panel t / 64 (i, j).
__device__ __forceinline__ double gram_colsums(GramStage& Ys, const double (&cs_i)[4], const double (&cs_j)[4], int panels)
{
    const int t = threadIdx.x, lrow = t >> 4, lcol = (t & 15) * 4;
    double* red = &Ys[0][0][0][0];                              // 2 x 16 x 64 doubles fit the first panel's two buffers
    static_assert(2 * kSdRows * kSdTile <= 2 * kSdRows * kSdPitch, "reduction scratch");
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        red[lrow * kSdTile + lcol + e] = cs_i[e];
        if (panels == 2) red[kSdRows * kSdTile + lrow * kSdTile + lcol + e] = cs_j[e];
    }
    __syncthreads();
    double v = 0.0;
    if (t < panels * kSdTile)
        for (int k = 0; k < kSdRows; ++k) v += red[(t >> 6) * kSdRows * kSdTile + k * kSdTile + (t & 63)];
    return v;
}

template <typename In>
__global__ void __launch_bounds__(256, 2)
stats_dmma_kernel(const In* __restrict__ E, const StatsDmmaParams p)
{
    __shared__ __align__(16) GramStage Ys;
    const int job = blockIdx.x;
    const int pair = job / p.n_splits, split = job % p.n_splits;
    int ti, tj;
    pair_to_tiles(pair, p.n_tiles, ti, tj);
    const long long row_begin = (long long)split * p.rows_per_split;
    const long long row_end = min(p.n_rows, row_begin + p.rows_per_split);
    double c[4][2][2] = {}, cs_i[4] = {0.0, 0.0, 0.0, 0.0}, cs_j[4] = {0.0, 0.0, 0.0, 0.0};
    gram_tile(Ys, E, p.d, row_begin, row_end, ti, tj, p.shift, c, cs_i, cs_j);
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
    const int fr = lane >> 2, fk = lane & 3;
    double* dst = p.ws_tiles + (size_t)job * kSdTile * kSdTile;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
            *reinterpret_cast<double2*>(dst + (wm + i * 8 + fr) * kSdTile + wn + j * 8 + 2 * fk) =
                make_double2(c[i][j][0], c[i][j][1]);
    if (ti == tj) {
        const double v = gram_colsums(Ys, cs_i, cs_j, 1);
        if (t < kSdTile) p.ws_sums[((size_t)ti * p.n_splits + split) * kSdTile + t] = v;
    }
}

// acc += sum over row splits of the job tiles, fixed order.  grid = (n_pairs, 16): block (pair, y) owns 256 of the
// tile's 4096 entries (a 3-block grid at d = 128 took 0.33 ms for 12 MB of partial tiles - longer than the Gram itself)
__global__ void __launch_bounds__(256) stats_dmma_reduce_kernel(StatsDmmaParams p, double* __restrict__ acc)
{
    const int pair = blockIdx.x;
    int ti, tj;
    pair_to_tiles(pair, p.n_tiles, ti, tj);
    const int d = p.d;
    double* outer = acc + 1 + d;
    {
        const int e = blockIdx.y * 256 + threadIdx.x;
        const int row = e / kSdTile, col = e % kSdTile;
        const double* src = p.ws_tiles + (size_t)pair * p.n_splits * kSdTile * kSdTile + e;
        double v0 = 0.0, v1 = 0.0, v2 = 0.0, v3 = 0.0;
        int s = 0;
        for (; s + 4 <= p.n_splits; s += 4) {                   // four loads in flight; the order of the sum stays fixed
            const double a = src[(size_t)(s + 0) * kSdTile * kSdTile], b = src[(size_t)(s + 1) * kSdTile * kSdTile];
            const double c = src[(size_t)(s + 2) * kSdTile * kSdTile], e4 = src[(size_t)(s + 3) * kSdTile * kSdTile];
            v0 += a; v1 += b; v2 += c; v3 += e4;
        }
        for (; s < p.n_splits; ++s) v0 += src[(size_t)s * kSdTile * kSdTile];
        const double v = (v0 + v1) + (v2 + v3);
        const int I = ti * kSdTile + row, J = tj * kSdTile + col;
        outer[(size_t)I * d + J] += v;
        if (ti != tj) outer[(size_t)J * d + I] += v;
    }
    if (ti == tj && blockIdx.y == 0) {
        for (int cidx = threadIdx.x; cidx < kSdTile; cidx += blockDim.x) {
            double v = 0.0;
            for (int s = 0; s < p.n_splits; ++s) v += p.ws_sums[((size_t)ti * p.n_splits + s) * kSdTile + cidx];
            acc[1 + ti * kSdTile + cidx] += v;                                        // sum(x - s), exact
            acc[1 + (size_t)d + (size_t)d * d + ti * kSdTile + cidx] += v;            // centring term: same y
        }
    }
    if (pair == 0 && blockIdx.y == 0 && threadIdx.x == 0) acc[0] += (double)p.n_rows;
}

// --------------------------------------------------------------------------------------
// Per-song statistics for fad_frechet_batched: item z owns rows [offsets[z], offsets[z+1]) of one fp16 [N, d] matrix.
// mean (rounded to fp16 like np.mean of an fp16 array, returned as fp64) and covariance (ddof = 1, exact fp64 products
// of y = x - s, s = the item's first row) of every item (fadtk/fad.py:42-48).  ok[z] = 0 for an item with fewer than 2
// rows (the reference asserts, fad.py:46): its covariance is set to the identity so the lock-step chain stays finite,
// and the assembly writes NaN.

// CUDA-core version, any d.  grid (ceil(d/32), ceil(d/32), items), 256 threads: thread (ty, tx) owns a 2 x 2 block.
__global__ void __launch_bounds__(256)
song_stats_kernel(const __half* __restrict__ emb, const long long* __restrict__ offsets, int d,
                  double* __restrict__ mu /*[items][d]*/, double* __restrict__ cov /*[items][d][d]*/,
                  int* __restrict__ ok)
{
    __shared__ double Yi[32][33], Yj[32][33];
    __shared__ double si[32], sj[32];
    const int z = blockIdx.z;
    const long long r0 = offsets[z], r1 = offsets[z + 1];
    const long long n = r1 - r0;
    const int bi = blockIdx.y * 32, bj = blockIdx.x * 32;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    double* C = cov + (size_t)z * d * d;
    if (n < 2) {
        for (int e = threadIdx.x; e < 1024; e += 256) {
            const int gi = bi + (e >> 5), gj = bj + (e & 31);
            if (gi < d && gj < d) C[(size_t)gi * d + gj] = gi == gj ? 1.0 : 0.0;
        }
        if (bj == 0 && threadIdx.x < 32 && bi + threadIdx.x < d) mu[(size_t)z * d + bi + threadIdx.x] = 0.0;
        if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) ok[z] = 0;
        return;
    }
    const __half* base = emb + (size_t)r0 * d;
    double c[2][2] = {};
    double colsum = 0.0;                                        // threads 0..31: column bi + t; 32..63: column bj + t
    for (long long rr = 0; rr < n; rr += 32) {
        for (int e = threadIdx.x; e < 2048; e += 256) {
            const int which = e >> 10, r = (e >> 5) & 31, cidx = e & 31;
            const int gc = (which ? bj : bi) + cidx;
            double v = 0.0;
            if (rr + r < n && gc < d)
                v = (double)__half2float(base[(size_t)(rr + r) * d + gc]) - (double)__half2float(base[gc]);
            (which ? Yj : Yi)[r][cidx] = v;
        }
        __syncthreads();
#pragma unroll 8
        for (int r = 0; r < 32; ++r) {
            const double a0 = Yi[r][ty * 2], a1 = Yi[r][ty * 2 + 1];
            const double b0 = Yj[r][tx * 2], b1 = Yj[r][tx * 2 + 1];
            c[0][0] = fma(a0, b0, c[0][0]); c[0][1] = fma(a0, b1, c[0][1]);
            c[1][0] = fma(a1, b0, c[1][0]); c[1][1] = fma(a1, b1, c[1][1]);
        }
        if (threadIdx.x < 64) {
            const int t = threadIdx.x & 31;
            double s = 0.0;
            if (threadIdx.x < 32) { for (int r = 0; r < 32; ++r) s += Yi[r][t]; }
            else                  { for (int r = 0; r < 32; ++r) s += Yj[r][t]; }
            colsum += s;
        }
        __syncthreads();
    }
    if (threadIdx.x < 32) si[threadIdx.x] = colsum;
    else if (threadIdx.x < 64) sj[threadIdx.x - 32] = colsum;
    __syncthreads();
    const double inv_n = 1.0 / (double)n, inv_n1 = 1.0 / (double)(n - 1);
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int v = 0; v < 2; ++v) {
            const int li = ty * 2 + u, lj = tx * 2 + v;
            const int gi = bi + li, gj = bj + lj;
            if (gi < d && gj < d) C[(size_t)gi * d + gj] = (c[u][v] - si[li] * sj[lj] * inv_n) * inv_n1;
        }
    if (bj == 0 && threadIdx.x < 32 && bi + threadIdx.x < d) {
        const double m = (double)__half2float(base[bi + threadIdx.x]) + si[threadIdx.x] * inv_n;
        mu[(size_t)z * d + bi + threadIdx.x] = (double)__half2float(__double2half(m));     // fp16 mean (fad.py:48)
    }
    if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) ok[z] = 1;
}

// The same statistics on the FP64 tensor pipe (d a multiple of 64): one CTA = (item, tile pair ti <= tj), the item's
// rows streamed through gram_tile, the covariance written to both triangles from the same accumulators.
// 5000 x [750, 128]: the CUDA-core kernel above was ~half of the whole per-song pass.  grid (n_pairs, items).
__global__ void __launch_bounds__(256, 2)
song_stats_dmma_kernel(const __half* __restrict__ emb, const long long* __restrict__ offsets, int d,
                       double* __restrict__ mu, double* __restrict__ cov, int* __restrict__ ok)
{
    constexpr int T = kSdTile;
    __shared__ __align__(16) GramStage Ys;
    __shared__ double s_sum[2][T];
    const int z = blockIdx.y;
    const long long n = offsets[z + 1] - offsets[z];
    int ti, tj;
    pair_to_tiles(blockIdx.x, d / T, ti, tj);
    const bool diag = ti == tj;
    const int t = threadIdx.x;
    double* C = cov + (size_t)z * d * d;
    if (n < 2) {
        for (int e = t; e < T * T; e += 256) {
            const int gi = ti * T + e / T, gj = tj * T + e % T;
            C[(size_t)gi * d + gj] = gi == gj ? 1.0 : 0.0;
            if (!diag) C[(size_t)gj * d + gi] = 0.0;
        }
        if (diag && t < T) mu[(size_t)z * d + ti * T + t] = 0.0;
        if (blockIdx.x == 0 && t == 0) ok[z] = 0;
        return;
    }
    const __half* base = emb + (size_t)offsets[z] * d;
    double c[4][2][2] = {}, cs_i[4] = {0.0, 0.0, 0.0, 0.0}, cs_j[4] = {0.0, 0.0, 0.0, 0.0};
    gram_tile(Ys, base, d, 0, n, ti, tj, base, c, cs_i, cs_j);
    const double sum = gram_colsums(Ys, cs_i, cs_j, 2);
    if (t < 2 * T) s_sum[t >> 6][t & 63] = sum;
    __syncthreads();
    const int warp = t >> 5, lane = t & 31;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
    const int fr = lane >> 2, fk = lane & 3;
    const double inv_n = 1.0 / (double)n, inv_n1 = 1.0 / (double)(n - 1);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int li = wm + i * 8 + fr, lj = wn + j * 8 + 2 * fk + e;
                const double v = (c[i][j][e] - s_sum[0][li] * s_sum[1][lj] * inv_n) * inv_n1;
                const int gi = ti * T + li, gj = tj * T + lj;
                C[(size_t)gi * d + gj] = v;
                if (!diag) C[(size_t)gj * d + gi] = v;
            }
    if (diag && t < T) {
        const double m = (double)__half2float(base[ti * T + t]) + s_sum[0][t] * inv_n;
        mu[(size_t)z * d + ti * T + t] = (double)__half2float(__double2half(m));      // fp16 mean (fad.py:48)
    }
    if (blockIdx.x == 0 && t == 0) ok[z] = 1;
}

// --------------------------------------------------------------------------------------
// fp64 CUDA-core version (verification path only: tensor_core = 2).  grid = (row chunks, d/64, d/64) upper tiles only.
constexpr int kSimtRows = 1024;
__global__ void __launch_bounds__(256)
stats_simt_kernel(const __half* __restrict__ E, long long n_rows, int d,
                  const __half* __restrict__ shift, double* __restrict__ acc)
{
    const int ti = blockIdx.y, tj = blockIdx.z;
    if (tj < ti) return;
    __shared__ double yi[32][65], yj[32][65];
    const long long r_begin = (long long)blockIdx.x * kSimtRows;
    const long long r_end = min(n_rows, r_begin + kSimtRows);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;      // 4x4 outputs per thread
    double c[4][4] = {};
    double csum = 0.0, csum_x = 0.0;
    for (long long r0 = r_begin; r0 < r_end; r0 += 32) {
        for (int i = threadIdx.x; i < 32 * 64; i += 256) {
            const int r = i >> 6, cc = i & 63;
            double a = 0.0, b = 0.0;
            if (r0 + r < r_end) {
                const __half* rowp = E + (size_t)(r0 + r) * d;
                // x - s in fp64 is exact for any two fp16 values; products of such differences carry
                // <= 2 x 40 bits, rounded once to fp64: relative error 1e-16 per term
                a = (double)__half2float(rowp[ti * 64 + cc]) - (double)__half2float(shift[ti * 64 + cc]);
                b = (double)__half2float(rowp[tj * 64 + cc]) - (double)__half2float(shift[tj * 64 + cc]);
            }
            yi[r][cc] = a; yj[r][cc] = b;
        }
        __syncthreads();
#pragma unroll 4
        for (int r = 0; r < 32; ++r) {
            double a[4], b[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { a[u] = yi[r][ty * 4 + u]; b[u] = yj[r][tx * 4 + u]; }
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) c[u][v] = fma(a[u], b[v], c[u][v]);
        }
        if (ti == tj && threadIdx.x < 64)
            for (int r = 0; r < 32; ++r) { csum += yi[r][threadIdx.x]; }
        csum_x = csum;                                      // y is exact here: both sums coincide
        __syncthreads();
    }
    double* outer = acc + 1 + d;
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int I = ti * 64 + ty * 4 + u, J = tj * 64 + tx * 4 + v;
            atomicAdd(&outer[(size_t)I * d + J], c[u][v]);
            if (ti != tj) atomicAdd(&outer[(size_t)J * d + I], c[u][v]);
        }
    if (ti == tj && threadIdx.x < 64) {
        atomicAdd(&acc[1 + ti * 64 + threadIdx.x], csum_x);
        atomicAdd(&acc[1 + (size_t)d + (size_t)d * d + ti * 64 + threadIdx.x], csum);
    }
    if (blockIdx.x == 0 && ti == 0 && tj == 0 && threadIdx.x == 0) atomicAdd(&acc[0], (double)n_rows);
}

// Per-file means of equal-length files (file f = rows [f r, (f + 1) r) of emb): the exact mean in fp64 and the mean as
// the reference's _process_file returns it for an fp16 .npy (np.mean of an fp16 array: fp32 accumulation, result rounded
// to fp16 - fadtk/utils.py:14), both stored as fp64 rows for the Gram kernel.  grid-stride over files x d.
__global__ void file_means_kernel(const __half* __restrict__ emb, long long n_files, int r, int d,
                                  double* __restrict__ m64, double* __restrict__ m16)
{
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n_files * d; e += (long long)gridDim.x * blockDim.x) {
        const long long f = e / d;
        const int c = (int)(e - f * d);
        const __half* src = emb + ((size_t)f * r) * d + c;
        double s64 = 0.0;
        float s32 = 0.f;
        for (int k = 0; k < r; ++k) { const float v = __half2float(src[(size_t)k * d]); s64 += (double)v; s32 += v; }
        m64[e] = s64 / (double)r;
        m16[e] = (double)__half2float(__float2half_rn(s32 / (float)r));
    }
}

// mu, cov as the reference's online merge computes them for n_files files of r rows each (fadtk/utils.py:13-46):
//   mu_ref = sum_f r m16_f / n,   S_ref = S_exact - sum_f r (m64_f - mu)(m64_f - mu)^T + sum_f r (m16_f - mu_ref)(m16_f - mu_ref)^T
// from the three packed accumulators (rows; exact file means; fp16-rounded file means - the latter two unshifted).
// r == 1 reproduces the reference's all-NaN covariance (np.cov of a single row) unless keep_single.
__global__ void stats_finalize_mirrored_kernel(const double* __restrict__ acc, const double* __restrict__ acc64,
                                               const double* __restrict__ acc16, const __half* __restrict__ shift,
                                               int r, int d, int keep_single, double* __restrict__ mu_out, double* __restrict__ cov_out)
{
    const double n = acc[0];
    const double* sum_x = acc + 1;
    const double* outer = acc + 1 + d;
    const double* sum_y = acc + 1 + (size_t)d + (size_t)d * d;
    const double* s64f = acc64 + 1;            // sum_f m64_f
    const double* o64 = acc64 + 1 + d;         // sum_f m64_f m64_f^T
    const double* s16f = acc16 + 1;
    const double* o16 = acc16 + 1 + d;
    const double w = (double)r;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)d * d; e += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(e / d), j = (int)(e % d);
        const double mu_i = (double)__half2float(shift[i]) + (n > 0.0 ? sum_x[i] / n : 0.0);
        const double mu_j = (double)__half2float(shift[j]) + (n > 0.0 ? sum_x[j] / n : 0.0);
        const double mr_i = n > 0.0 ? w * s16f[i] / n : 0.0, mr_j = n > 0.0 ? w * s16f[j] / n : 0.0;
        double c = 0.0;
        if (n >= 2.0) {
            const double s_exact = outer[e] - sum_y[i] * sum_y[j] / n;                               // (n - 1) cov_exact
            const double b64 = w * o64[e] - mu_i * (w * s64f[j]) - (w * s64f[i]) * mu_j + n * mu_i * mu_j;
            const double b16 = w * o16[e] - mr_i * (w * s16f[j]) - (w * s16f[i]) * mr_j + n * mr_i * mr_j;
            c = (s_exact - b64 + b16) / (n - 1.0);
            if (r == 1 && !keep_single) c = nan;
        }
        cov_out[e] = c;
        if (j == 0) mu_out[i] = mr_i;
    }
}

// mu = shift + sum(x-s)/n ; cov = (outer - sum(y) sum(y)^T / n) / (n - 1)   (cov = 0 when n < 2,
// fadtk/utils.py:42-43).  grid-stride over d*d.
__global__ void stats_finalize_kernel(const double* __restrict__ acc, const __half* __restrict__ shift,
                                      int d, double* __restrict__ mu, double* __restrict__ cov)
{
    const double n = acc[0];
    const double* sum_x = acc + 1;
    const double* outer = acc + 1 + d;
    const double* sum = acc + 1 + (size_t)d + (size_t)d * d;
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)d * d;
         e += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(e / d), j = (int)(e % d);
        cov[e] = n < 2.0 ? 0.0 : (outer[e] - sum[i] * sum[j] / n) / (n - 1.0);
        if (j == 0) mu[i] = (double)__half2float(shift[i]) + (n > 0.0 ? sum_x[i] / n : 0.0);
    }
}

// out[i, :] = src[idx[i], :]  (FAD-inf bootstrap gather, fadtk/fad.py:333-334); 16-B vectors.
__global__ void gather_rows_kernel(const __half* __restrict__ src, const long long* __restrict__ idx,
                                   long long n_out, int d, __half* __restrict__ out)
{
    const int vec_per_row = d / 8;
    const long long total = n_out * vec_per_row;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long i = e / vec_per_row;
        const int v = (int)(e % vec_per_row);
        reinterpret_cast<uint4*>(out)[e] = reinterpret_cast<const uint4*>(src + (size_t)idx[i] * d)[v];
    }
}

// --------------------------------------------------------------------------------------
// Permutation test of the FAD difference between two systems (DESIGN.md 5.17).  A unit is one file: rows
// [offsets[u], offsets[u + 1]) of one fp16 [N, d] pool, d a multiple of 64.  Its record is
//   R_u = [n_u | sum y (d) | upper triangle of sum y y^T, row by row (d (d + 1) / 2)],   y = x - s,
// s the fp16 shift of the pool.  Every product of two fp16 differences is exact in fp64, so a record carries only the
// fp64 summation rounding of gram_tile.  Records add: the statistics of a union of units are the sum of their records.
__host__ __device__ constexpr long long record_len(int d) { return 1 + (long long)d + (long long)d * (d + 1) / 2; }
// packed position of (I, J), I <= J, in the upper triangle
__device__ __forceinline__ long long record_upper(int d, int I, int J) {
    return (long long)I * d - (long long)I * (I - 1) / 2 + (J - I);
}

// records[u] of the units u of this launch (offsets: absolute rows of its first unit onwards).  One CTA = (tile pair
// ti <= tj, unit) as song_stats_dmma_kernel; the diagonal tiles also write sum y, tile pair 0 writes n.
// grid (n_pairs, units).
__global__ void __launch_bounds__(256, 2)
unit_records_kernel(const __half* __restrict__ emb, const long long* __restrict__ offsets, int d,
                    const __half* __restrict__ shift, double* __restrict__ records)
{
    constexpr int T = kSdTile;
    __shared__ __align__(16) GramStage Ys;
    const long long r0 = offsets[blockIdx.y], r1 = offsets[blockIdx.y + 1];
    int ti, tj;
    pair_to_tiles(blockIdx.x, d / T, ti, tj);
    double* rec = records + (size_t)blockIdx.y * record_len(d);
    double c[4][2][2] = {}, cs_i[4] = {0.0, 0.0, 0.0, 0.0}, cs_j[4] = {0.0, 0.0, 0.0, 0.0};
    gram_tile(Ys, emb, d, r0, r1, ti, tj, shift, c, cs_i, cs_j);
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
    const int fr = lane >> 2, fk = lane & 3;
    double* upper = rec + 1 + d;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int I = ti * T + wm + i * 8 + fr, J = tj * T + wn + j * 8 + 2 * fk + e;
                if (I <= J) upper[record_upper(d, I, J)] = c[i][j][e];
            }
    if (ti == tj) {
        const double v = gram_colsums(Ys, cs_i, cs_j, 1);
        if (t < T) rec[1 + ti * T + t] = v;
    }
    if (blockIdx.x == 0 && t == 0) rec[0] = (double)(r1 - r0);
}

// Labelled record sums: for every labelling b of the launch and both sides,
//   sums[b][0] += sum_u l_b(u) R_u,   sums[b][1] += sum_u (1 - l_b(u)) R_u
// as a GEMM on the FP64 tensor pipe (mma.sync m8n8k4 f64): M = labellings, N = record columns, K = units.  The labels
// of a k-step are expanded from the bits (fad_perm_labels' layout) to fp64 0 / 1 in registers, the A operand of both
// sides; the B operand (16 units x 64 columns of records) is staged in shared memory as in dgemm_tile.  Each
// accumulator element runs the units in order, four per DMMA, from zero or from the value a previous launch stored:
// when every launch but the last covers a multiple of 4 units (the host uses multiples of 64), the result is bitwise
// the same however the units are cut into launches and the labellings into passes.  No atomics.
//
// kWeighted (the bootstrap, DESIGN.md 5.18): sums[b] += sum_u w_b(u) R_u, one accumulator, the A operand the integer
// multiplicities w_b(u) of the launch's units (counts: [rows][count_stride], column 0 = the launch's first unit)
// converted to fp64 in registers, exactly.  Same staging, order and invariance; bits and words are not read.
constexpr int kRsTile = 64, kRsUnits = 16, kRsPitch = kRsTile + 4;
constexpr int kRsUnitAlign = 64;                  // unit0 of every launch is a multiple of this

struct RecordSumsParams {
    const double* records;       // [units][R]: the launch's units
    long long R;
    int units, unit0;            // units of this launch; the first one's index in the pool (label bit position)
    const uint32_t* bits;        // labelling 0 of this launch
    int words;                   // words per labelling
    int rows;                    // labellings of this launch: rows past it are not read nor written
    int accumulate;              // 0: start from zero, 1: add to sums
    double* sums;                // [rows][2][R]; kWeighted: [rows][R]
    const uint32_t* counts;      // kWeighted: multiplicities [rows][count_stride] of the launch's units
    long long count_stride;
};

template <bool kWeighted>
__global__ void __launch_bounds__(256, 1)
record_sums_kernel(const RecordSumsParams p)
{
    __shared__ __align__(16) double Rs[2][kRsUnits][kRsPitch];
    const int m0 = blockIdx.x * kRsTile;
    const long long n0 = (long long)blockIdx.y * kRsTile;
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
    const int fr = lane >> 2, fk = lane & 3;
    const int lu = t >> 4, lc = (t & 15) * 4;                   // loader: unit of the stage, first of 4 columns
    const long long R = p.R;

    double ca[4][2][2], cb[4][2][2];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int m = m0 + wm + i * 8 + fr;
                const long long n = n0 + wn + j * 8 + 2 * fk + e;
                const bool in = p.accumulate && m < p.rows && n < R;
                if constexpr (kWeighted) {
                    ca[i][j][e] = in ? p.sums[(size_t)m * R + n] : 0.0;
                } else {
                    ca[i][j][e] = in ? p.sums[((size_t)m * 2) * R + n] : 0.0;
                    cb[i][j][e] = in ? p.sums[((size_t)m * 2 + 1) * R + n] : 0.0;
                }
            }
    const int mrow = m0 + wm + fr;                               // this thread's labelling rows: mrow + 8 i
    const uint32_t* lb = p.bits + (size_t)mrow * p.words;

    double rv[4];
    auto fetch = [&](int st) {
        const int u = st * kRsUnits + lu;
        const double* src = p.records + (size_t)u * R + n0 + lc;
#pragma unroll
        for (int e = 0; e < 4; ++e) rv[e] = (u < p.units && n0 + lc + e < R) ? __ldg(src + e) : 0.0;
    };
    auto stage = [&](int buf) {
        *reinterpret_cast<double2*>(&Rs[buf][lu][lc]) = make_double2(rv[0], rv[1]);
        *reinterpret_cast<double2*>(&Rs[buf][lu][lc + 2]) = make_double2(rv[2], rv[3]);
    };
    const int stages = (p.units + kRsUnits - 1) / kRsUnits;
    fetch(0);
    stage(0);
    __syncthreads();
    for (int st = 0; st < stages; ++st) {
        const int buf = st & 1;
        if (st + 1 < stages) fetch(st + 1);
        if constexpr (kWeighted) {
            const uint32_t* cnt = p.counts + (size_t)mrow * p.count_stride + st * kRsUnits + fk;
#pragma unroll
            for (int kk = 0; kk < kRsUnits; kk += 4) {
                const bool valid = st * kRsUnits + kk + fk < p.units;
                double b[2];
#pragma unroll
                for (int j = 0; j < 2; ++j) b[j] = Rs[buf][kk + fk][wn + j * 8 + fr];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const double a = valid && mrow + 8 * i < p.rows
                        ? (double)__ldg(cnt + (size_t)8 * i * p.count_stride + kk) : 0.0;
#pragma unroll
                    for (int j = 0; j < 2; ++j) sm90::dmma_884(ca[i][j][0], ca[i][j][1], a, b[j]);
                }
            }
            if (st + 1 < stages) stage(buf ^ 1);
            __syncthreads();
            continue;
        }
        const int ug = p.unit0 + st * kRsUnits;                  // a multiple of 16: the stage sits in one word
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
            w[i] = mrow + 8 * i < p.rows ? __ldg(lb + (size_t)8 * i * p.words + (ug >> 5)) >> (ug & 31) : 0u;
#pragma unroll
        for (int kk = 0; kk < kRsUnits; kk += 4) {
            const bool valid = st * kRsUnits + kk + fk < p.units;
            double b[2];
#pragma unroll
            for (int j = 0; j < 2; ++j) b[j] = Rs[buf][kk + fk][wn + j * 8 + fr];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const uint32_t bit = (w[i] >> (kk + fk)) & 1u;
                const double a = valid && bit ? 1.0 : 0.0, ac = valid && !bit ? 1.0 : 0.0;
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    sm90::dmma_884(ca[i][j][0], ca[i][j][1], a, b[j]);
                    sm90::dmma_884(cb[i][j][0], cb[i][j][1], ac, b[j]);
                }
            }
        }
        if (st + 1 < stages) stage(buf ^ 1);
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int m = m0 + wm + i * 8 + fr;
                const long long n = n0 + wn + j * 8 + 2 * fk + e;
                if constexpr (kWeighted) {
                    if (m < p.rows && n < R) p.sums[(size_t)m * R + n] = ca[i][j][e];
                } else if (m < p.rows && n < R) {
                    p.sums[((size_t)m * 2) * R + n] = ca[i][j][e];
                    p.sums[((size_t)m * 2 + 1) * R + n] = cb[i][j][e];
                }
            }
}

// Item z of a Frechet group from its labelled sum S = sums + z R: mu = s + sum y / n (fp64), the symmetric
// C = (sum y y^T - sum y sum y^T / n) / (n - 1), ok[z], and n into out[z][7].  An item with n < 2 gets the identity
// and ok = 0 as in song_stats_kernel (the assembly writes NaN).  grid (blocks, items).
__global__ void __launch_bounds__(256)
record_finalize_kernel(const double* __restrict__ sums, int d, const __half* __restrict__ shift,
                       double* __restrict__ mu, double* __restrict__ cov, int* __restrict__ ok, double* __restrict__ out)
{
    const int z = blockIdx.y;
    const double* S = sums + (size_t)z * record_len(d);
    const double n = S[0];
    const double* sy = S + 1;
    const double* upper = S + 1 + d;
    const bool good = n >= 2.0;
    double* C = cov + (size_t)z * d * d;
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)d * d; e += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(e / d), j = (int)(e % d);
        C[e] = good ? (upper[record_upper(d, min(i, j), max(i, j))] - sy[i] * sy[j] / n) / (n - 1.0) : (i == j ? 1.0 : 0.0);
        if (j == 0) mu[(size_t)z * d + i] = good ? (double)__half2float(shift[i]) + sy[i] / n : 0.0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        ok[z] = good ? 1 : 0;
        out[(size_t)z * 8 + 7] = n;
    }
}

}  // namespace fad
