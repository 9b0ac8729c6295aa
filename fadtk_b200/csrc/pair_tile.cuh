// The pair-tile device code both pairwise metrics run, Kernel Audio Distance (kad.cuh) and precision, recall, density
// and coverage (prdc.cuh): the prologue that shifts, splits and takes the norms of the rows of Z, the TMA + wgmma tile
// loop that turns two 128-row boxes of Z into the fp32 dot products of their rows, the one formula for the squared
// distance q of a pair, the song map of the per-song passes, and the digest and shard sum of a sharded call.
//
// Precision.  q = |z_i|^2 + |z_j|^2 - 2 z_i.z_j cancels: rows with a large common offset (Encodec: |mu| ~ 64 per
// dimension, spread ~ 2) have norms ~1000 x the distances, and an fp32 dot product then leaves ~1e-4 relative error in
// q.  So a prologue (pair_split_kernel) subtracts a shift s shared by all rows (the fp16-rounded mean of X; distances
// do not depend on it), and splits y = z - s (exact in fp32) into an fp16 pair hi + lo (22 bits).  The tile loop
// issues hi.hi + hi.lo + lo.hi per k-step into one fp32 accumulator (lo.lo is 2^-22 of the result and dropped).  Row
// norms are the same three terms in fp64, rounded to fp32 once, so an identical pair of rows gives q = 0 up to the
// accumulator's rounding; q below kQResolution * (|y_i|^2 + |y_j|^2), the resolution of the expanded form, is taken as
// 0 (pair_q; exact duplicates have q = 0: silent clips, sigma = 0 detection).  The accumulator uses the GEMM's
// chunk-and-unshrink scheme (conv_gemm.cuh), counting the three products per column.
//
// Warp roles (384 threads, persistent): warpgroup 0 = TMA producer (one elected lane); warpgroups 1-2 = consumers,
// consumer c owns tile rows [64 c, 64 c + 64) x 128 columns (one m64n128 accumulator), issues the wgmmas and runs its
// kernel's epilogue on the accumulator fragment in its registers - no shared-memory round trip of the tile.  Stage =
// {A_hi, A_lo, B_hi, B_lo} boxes of 128 rows x 64 columns (64 KiB), 3 stages.
#pragma once
#include "sm90.cuh"
#include "conv_gemm.cuh"

namespace fad {

constexpr int kPairThreads = 384;
constexpr int kPairStages = 3;
constexpr int kPairConsumerRegs = 232;              // 40 x 128 + 232 x 256 <= 65536
constexpr uint32_t kPairBox = 128 * 64 * 2;         // one 128-row x 64-column fp16 box (16 KiB)
constexpr uint32_t kPairStageBytes = 4 * kPairBox;  // A_hi, A_lo, B_hi, B_lo
// the stages, the 1024-byte alignment slack and the barriers; a kernel's own shared memory follows (pair_tile_open)
constexpr uint32_t kPairSmemBytes = kPairStages * kPairStageBytes + 1024 + 256;
// q below this fraction of |y_i|^2 + |y_j|^2 is not resolved by the expanded form in fp32 (worst-case accumulator
// rounding at d = 1024 is ~2e-5 of it) and is taken as 0
constexpr float kQResolution = 6.103515625e-05f;    // 2^-14
constexpr int kPairColRows = 4096;                  // rows per partial column sum of the shift prologue
static_assert(40 * 128 + kPairConsumerRegs * 256 <= 65536, "register file over-subscribed");

// --------------------------------------------------------------------------------------------- prologue
// part[chunk][col] = sum of z[r][col] over the rows of chunk (fp64, fixed order)
__global__ void pair_colsum_kernel(const __half* __restrict__ z, int m, int d, double* __restrict__ part) {
    const int r0 = blockIdx.x * kPairColRows;
    const int r1 = min(m, r0 + kPairColRows);
    for (int col = threadIdx.x; col < d; col += blockDim.x) {
        double s = 0.0;
        for (int r = r0; r < r1; ++r) s += (double)__half2float(z[(size_t)r * d + col]);
        part[(size_t)blockIdx.x * d + col] = s;
    }
}
// shift = fp16(mean of the first m rows), the partial sums added in chunk order
__global__ void pair_shift_kernel(const double* __restrict__ part, int chunks, int m, int d, __half* __restrict__ shift) {
    for (int col = threadIdx.x; col < d; col += blockDim.x) {
        double s = 0.0;
        for (int c = 0; c < chunks; ++c) s += part[(size_t)c * d + col];
        shift[col] = __double2half(s / (double)m);
    }
}
// one warp per row: y = z - shift (exact in fp32), hi = fp16(y), lo = fp16(y - hi); norm = sum hi^2 + 2 hi lo (fp64,
// fixed lane order, then a fixed shuffle tree), the terms the tile loop's dot products contain
__global__ void pair_split_kernel(const __half* __restrict__ z, int N, int rows_pad, int d, const __half* __restrict__ shift,
                                  __half* __restrict__ hi, __half* __restrict__ lo, float* __restrict__ norm) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows_pad) return;
    double acc = 0.0;
    if (row < N) {
        for (int col = lane; col < d; col += 32) {
            const size_t e = (size_t)row * d + col;
            const float y = __half2float(z[e]) - __half2float(shift[col]);
            const __half h = __float2half_rn(y);
            const __half l = __float2half_rn(y - __half2float(h));
            hi[e] = h;
            lo[e] = l;
            const double hd = (double)__half2float(h), ld = (double)__half2float(l);
            acc += hd * hd + 2.0 * hd * ld;
        }
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) norm[row] = (float)acc;
}

// per-song passes: song_of[r] for the Y rows r < rows = the song s with offsets[s] <= r < offsets[s + 1]; -1 from n_total
__global__ void pair_song_of_kernel(const long long* __restrict__ offsets, long long n_items, long long n_total, int rows,
                                    int* __restrict__ song_of) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    if (r >= n_total) { song_of[r] = -1; return; }
    long long lo = 0, hi = n_items;                 // offsets[lo] <= r < offsets[hi]
    while (hi - lo > 1) {
        const long long mid = (lo + hi) >> 1;
        if (offsets[mid] <= r) lo = mid; else hi = mid;
    }
    song_of[r] = (int)lo;
}

// ------------------------------------------------------------------------------------------- tile loop
// The opening of a tile kernel: the stages at the 1024-aligned start of dynamic shared memory, the full / empty barriers
// after them (thread 0 prefetches the two descriptors and initialises the barriers), and the k-steps of d cut into
// near-equal accumulation chunks.  own = the kernel's own shared memory; the kernel clears what it needs, then
// __syncthreads().
struct PairTile {
    uint8_t* smem;
    uint64_t* full;
    uint64_t* empty;
    uint8_t* own;
    int ksteps, chunk_len;
};
__device__ __forceinline__ PairTile pair_tile_open(uint8_t* smem_raw, const CUtensorMap* map_hi, const CUtensorMap* map_lo,
                                                   int d, int warp, int lane) {
    using namespace sm90;
    PairTile t;
    t.smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    t.full = reinterpret_cast<uint64_t*>(t.smem + kPairStages * kPairStageBytes);
    t.empty = t.full + kPairStages;
    t.own = t.smem + kPairStages * kPairStageBytes + 256;
    t.ksteps = (d + 63) / 64;
    const int n_chunks = (t.ksteps + kChunkSteps - 1) / kChunkSteps;
    t.chunk_len = (t.ksteps + n_chunks - 1) / n_chunks;
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(map_hi);
        tma_prefetch_desc(map_lo);
        for (int s = 0; s < kPairStages; ++s) { mbar_init(&t.full[s], 1); mbar_init(&t.empty[s], 8); }   // 8 consumer warps
        mbar_fence_init();
    }
    return t;
}

// producer: the ksteps stages of one tile, A = rows [arow, arow + 128), B = rows [brow, brow + 128) of Z (rows past N
// are zero-filled by the TMA unit; neither coordinate needs to be a multiple of 128)
__device__ __forceinline__ void pair_load_tile(uint8_t* smem, uint64_t* full, uint64_t* empty, int& s, uint32_t& ph,
                                               const CUtensorMap* map_hi, const CUtensorMap* map_lo, int ksteps,
                                               int arow, int brow) {
    using namespace sm90;
    for (int ks = 0; ks < ksteps; ++ks) {
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = smem + s * kPairStageBytes;
        mbar_expect_tx(&full[s], kPairStageBytes);
        tma_load_2d(st, map_hi, &full[s], ks * 64, arow);
        tma_load_2d(st + kPairBox, map_lo, &full[s], ks * 64, arow);
        tma_load_2d(st + 2 * kPairBox, map_hi, &full[s], ks * 64, brow);
        tma_load_2d(st + 3 * kPairBox, map_lo, &full[s], ks * 64, brow);
        if (++s == kPairStages) { s = 0; ph ^= 1; }
    }
}

// consumer c: sum = the fp32 dot products y_i.y_j (hi.hi + hi.lo + lo.hi) of its 64 x 128 block of one tile, in the
// m64n128 fragment layout: element (tile row 64 c + 16 (warp & 3) + (lane >> 2) + 8 i, tile column 2 (lane & 3) + 8 j + e)
// is sum[4 j + 2 i + e]
__device__ __forceinline__ void pair_mma_tile(float (&sum)[64], uint8_t* smem, uint64_t* full, uint64_t* empty, int& s,
                                              uint32_t& ph, int c, int lane, int d, int ksteps, int chunk_len) {
    using namespace sm90;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) sum[i] = 0.f;
    for (int ks0 = 0; ks0 < ksteps; ks0 += chunk_len) {
        const int ks1 = min(ks0 + chunk_len, ksteps);
        // three products per real column accumulate into each element (zero-filled columns add exact zeros, which do
        // not truncate)
        const int cols = min(d, ks1 * 64) - ks0 * 64;
        const float unshrink = kAccumShrinkPerElement * (float)(3 * cols);
        int prev_s = -1;
        for (int ks = ks0; ks < ks1; ++ks) {
            mbar_wait(&full[s], ph);
            const uint32_t base = smem_u32(smem + s * kPairStageBytes);
            const uint64_t ah = kmajor_sw128_desc(base + c * 64 * 128);
            const uint64_t al = kmajor_sw128_desc(base + kPairBox + c * 64 * 128);
            const uint64_t bh = kmajor_sw128_desc(base + 2 * kPairBox);
            const uint64_t bl = kmajor_sw128_desc(base + 3 * kPairBox);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                wgmma_m64n128k16_f16<0, 0>(acc, ah + 2 * k, bh + 2 * k, (ks > ks0) || (k > 0));
                wgmma_m64n128k16_f16<0, 0>(acc, ah + 2 * k, bl + 2 * k, 1);
                wgmma_m64n128k16_f16<0, 0>(acc, al + 2 * k, bh + 2 * k, 1);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (prev_s >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev_s]); }
            prev_s = s;
            if (++s == kPairStages) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev_s]);
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] += fmaf(acc[i], unshrink, acc[i]);
    }
}

// the squared distance of a pair from its dot product and the two row norms; below the resolution (also q < 0): 0
__device__ __forceinline__ float pair_q(float dot, float nr, float nc) {
    const float sn = nr + nc;
    const float q = fmaf(-2.f, dot, sn);
    return q > kQResolution * sn ? q : 0.f;
}

// ------------------------------------------------------------------------------------------- sharding
// sharded passes (pairwise_host.inc, exchange): buf[i] = buf[i] + buf[n + i] + ... over the shards' copies in shard
// order.  Each value is written by one shard and zero in the others, so the sum is that value exactly.
template <typename T>
__global__ void pair_shard_sum_kernel(T* __restrict__ buf, long long n, int shards) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        T s = buf[i];
        for (int c = 1; c < shards; ++c) s += buf[(size_t)c * n + i];
        buf[i] = s;
    }
}

// *out += the wrapping sum over the 16-bit elements of z, read as n_vec words W (uint4: 8 elements, uint32_t: 2), of a
// 64-bit mix of (element index, element bits): an order-independent digest the ranks of a sharded call compare before
// any tile work.  uint4 for the fp16 rows; uint32_t for fp32 arrays, which are only 4-byte aligned and need not fill
// a whole number of uint4.
__host__ __device__ __forceinline__ unsigned long long pair_mix64(unsigned long long x) {   // splitmix64 finaliser
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
template <typename W>
__global__ void pair_digest_kernel(const W* __restrict__ z, long long n_vec, unsigned long long* __restrict__ out) {
    constexpr int kElems = sizeof(W) / 2;
    unsigned long long s = 0;
    for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < n_vec; v += (long long)gridDim.x * blockDim.x) {
        const W q = z[v];
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&q);
#pragma unroll
        for (int k = 0; k < kElems; ++k) {
            const unsigned long long e = (unsigned long long)(kElems * v + k);
            s += pair_mix64((e << 16) | ((w[k >> 1] >> (16 * (k & 1))) & 0xFFFFu));
        }
    }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(out, s);
}

}  // namespace fad
