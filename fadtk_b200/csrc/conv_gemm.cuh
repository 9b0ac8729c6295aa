// Implicit-GEMM 3x3 convolution / fully-connected layer on Hopper tensor cores (wgmma).
//
//   D[128 pixels, N_TILE channels] = sum over (tap, 64-channel block) of
//         X_tap[128 pixels, 64 ch] (fp16, K-major, TMA im2col-by-coordinates)
//       x W[N_TILE, (tap, 64 ch)]^T (fp16, K-major)
//   epilogue: + bias, ReLU, optional 2x2 max-pool, fp32 -> fp16, NHWC store.
//
// Replaces the cuDNN / cuBLAS calls behind torchvggish's ``features`` and ``embeddings``
// (reference call site fadtk/model_loader.py:107-108; shapes in SURVEY.md appendix A, K3/K4).
//
// Data movement: activations are NHWC fp16 in HBM.  One output tile covers a
// BW x BH x BN box of pixels (BW*BH*BN = 128); for filter tap (kh, kw) the A operand is the
// same box shifted by (kh-1, kw-1), fetched with ONE 4-D TMA whose out-of-bounds elements are
// zero-filled by hardware - that is the conv padding, and there is no im2col buffer.  TMA
// writes the 128-byte swizzled K-major layout wgmma consumes directly.
//
// Accumulation.  The tensor core adds into its fp32 accumulator with truncation, so a long K
// reduction comes out slightly shrunk (tests/diag_accum_bias.py measures it).  So each consumer
// warpgroup accumulates at most kChunkSteps x 64 = 512 of K into its wgmma accumulator, then adds
// the chunk into a second register array with ordinary round-to-nearest fp32 adds.
//
// Warp roles (512 threads, persistent over tiles; every role walks the same sequence of work units):
//   warpgroup 0     TMA producer (one elected lane of warp 0)
//   warpgroups 1-2  consumers: warpgroup 1 + c issues the wgmmas of tile rows [64 c, 64 c + 64), folds the chunks,
//                   dumps the finished accumulator into its half of the fp32 shared-memory tile and starts the next
//                   tile at once
//   warpgroup 3     epilogue: warps 2 c and 2 c + 1 drain consumer c's half (32 rows each, one row per lane): bias,
//                   activation, pool, stores, fused residual - overlapped with the consumers' next main loop
// Pipeline: smem ring full[] (TMA -> consumers) / empty[] (consumers -> TMA); per consumer half, epi_full[c]
// (consumer -> epilogue) / epi_empty[c] (epilogue -> consumer).  The handoff is per half, so one never waits for
// the other.  Registers per thread (setmaxnreg): producer 40, epilogue kEpiRegs, consumers kConsumerRegs
// (40 + 136 + 2 x 168 = 512 = 65536 / 128): a consumer holds sum[64] + acc[64] + addressing, nothing of the epilogue;
// the epilogue walks its row 32 columns at a time.  ptxas -v: no spills in either instantiation.
//
// CTA pairs.  The kernel runs in clusters of two CTAs; the work unit is (pair of neighbouring M tiles, N tile) and
// cluster rank r computes M tile 2 mp + r.  Both tiles need the same weight box at every k-step, so each rank loads
// half of its rows (split weights: rank 0 the hi rows, rank 1 the lo rows) and multicasts them into the same stage of
// both CTAs: per CTA and k-step, 16 KiB of weights come from L2 instead of 32 (16 KiB + 8 KiB instead of 16 + 16 with
// fp16 weights).  A stage is refilled only when the consumers of BOTH CTAs are done with it.  With an odd number of M
// tiles the last pair's rank 1 is a spare: it loads its weight half and runs the pipeline on rank 0's A rows, and its
// epilogue stores nothing (its rows are all >= NB).  Every tile runs the same wgmma sequence as with one CTA per tile.
#pragma once
#include "sm90.cuh"

namespace fad {

struct ConvGemmParams {
    int taps;        // 9 (conv3x3, pad 1) or 1 (fully connected / 1x1)
    int cblks;       // Cin / 64
    int box_w, box_h, box_n;   // pixel box of one tile, product == 128
    int tiles_w, tiles_h;      // tiles per image along W and H
    int img_groups;            // ceil(NB / box_n)
    int n_tiles;               // Cout / N_TILE
    int H, W, NB, Cout;
    int lo_adds;               // WMODE 1: 1 = the lo parts are not all zero, so their wgmmas truncate the accumulator too
    int ld_out, n_valid;       // un-pooled outputs: row stride and number of columns actually stored
                               // (Cout is padded to the tile width; columns >= n_valid are dropped)
    int relu, pool;            // relu: 0 = none, 1 = ReLU, 2 = GELU (erf form), 3 = ELU
    const float* bias;         // [Cout]
    __half* out;               // NHWC fp16 [NB, H(/2), W(/2), Cout]; may be null when out_f32 is set
    float* out_f32;            // optional fp32 copy of the un-pooled output (may be null)
    // optional fused residual update (transformer blocks): resid[token(row)][0:resid_C] += result,
    // where row -> token undoes the (shifted-)window ordering of the rows (resid_res = 0: identity)
    float* resid;
    int resid_C, resid_res, resid_shift;
};

// token index (b*res*res + y*res + x) of window-ordered row o (8x8 windows, cyclic shift)
__device__ __forceinline__ long long window_row_to_token(long long o, int res, int shift) {
    const int lg_nw = 28 - __clz(res);                 // res is a power of two >= 8: log2(res / 8)
    const int nw = res >> 3;
    const int in = (int)(o & 63);
    const long long wi = o >> 6;
    const int wx = (int)wi & (nw - 1);
    const int wy = (int)(wi >> lg_nw) & (nw - 1);
    const long long b = wi >> (2 * lg_nw);
    int y = wy * 8 + (in >> 3) + shift, xx = wx * 8 + (in & 7) + shift;
    if (y >= res) y -= res;
    if (xx >= res) xx -= res;
    return (b * res + y) * res + xx;
}

constexpr int kTileM = 128;
constexpr int kBlockK = 64;                        // fp16 elements per 128-B swizzled row
constexpr int kConvGemmThreads = 512;
constexpr int kConsumers = 2;                      // consumer warpgroups, 64 tile rows each
constexpr int kConsumerRegs = 168;                 // setmaxnreg budgets: 40 + kEpiRegs + 2 x kConsumerRegs <= 512
constexpr int kEpiRegs = 136;
constexpr int kClusterCtas = 2;                    // CTAs per cluster, sharing each weight box
constexpr int kChunkSteps = 8;                     // k-steps (of 64) per accumulation chunk
// The tensor core truncates when it adds into its fp32 accumulator: a sum over T accumulated elements (T = K of the
// chunk) comes out scaled by (1 - c T), c = 1.06e-9 measured on H100 with tests/diag_accum_bias.py.  Cutting K into
// chunks bounds it, but what is left is SYSTEMATIC: through the ~50 GEMMs of a transformer encoder it adds up to a
// per-dimension offset of the hidden states and of the FAD.  The consumer therefore scales every chunk by the inverse
// of its expected shrink when it sums the chunks in registers: v + v * eps as one FMA (1 + eps itself is not
// representable finely enough in fp32: eps ~ 1e-6 is only 8 ulps of 1).  c is what tests/diag_accum_bias.py measures.
constexpr float kAccumShrinkPerElement = 1.06e-9f;
constexpr uint32_t kABytes = kTileM * kBlockK * 2; // 16 KiB per stage
constexpr uint32_t kEpiRowBytes = 128 * 4;         // one fp32 row of a 128-column accumulator tile
constexpr uint32_t kEpiBytes = 64 * kEpiRowBytes;  // per consumer: 64 rows x 128 fp32 (32 KiB)
constexpr uint32_t kBiasBytes = 128 * 4;           // per epilogue warp: the bias of the tile's 128 columns
static_assert(40 + kEpiRegs + kConsumers * kConsumerRegs <= 65536 / 128, "register file over-subscribed");
static_assert(kConsumerRegs > 65536 / kConvGemmThreads, "the consumers raise their register count (setmaxnreg.inc)");

// SPLIT_W: the weights are an fp16 hi/lo pair (W = Wh + Wl, 22 bits).  fp16 rounding of the
// weights is a fixed perturbation of the model that does not average out over samples: it alone
// moves the FAD by ~1.4e-4 relative (CPU experiment, DESIGN.md), more than the whole 1e-4 budget,
// whereas fp16 activations cost 2e-5.  The hi and lo rows of one N tile are stored back to back
// ([Wh: N_TILE rows | Wl: N_TILE rows] per tile), so ONE TMA box brings both and each consumer
// issues A x Wh and A x Wl into the same accumulator.
// WMODE 0: fp16 weights, one wgmma per K slice.  WMODE 1: fp16 hi/lo pair (SPLIT_W), two fp16
// wgmmas per K slice into one accumulator.
template <int N_TILE, int WMODE>
__host__ __device__ constexpr uint32_t conv_gemm_stage_bytes() {
    return kABytes + (WMODE == 1 ? 2 : 1) * N_TILE * kBlockK * 2;
}

template <int N_TILE, int STAGES, int WMODE>
__host__ __device__ constexpr uint32_t conv_gemm_smem_bytes() {
    return STAGES * conv_gemm_stage_bytes<N_TILE, WMODE>() + 1024 /*align slack*/ + 256 /*barriers*/
         + kConsumers * kEpiBytes + 4 * kBiasBytes;
}

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&h);
}
// GELU(x) = x/2 (1 + erf(x / sqrt 2)), the exact-erf form torch.nn.GELU() / HTSAT use, with
//   erf(z) = 1 - 2^(z q(z)),  z = |x| / sqrt 2 clamped to 4.3   (erfc(4.3) = 1.2e-9)
// q = degree-6 weighted-minimax fit of log2(erfc(z)) / z (oracle/fit_gelu.py): |erf error| <= 1.4e-7
// in fp32, far below the fp16 rounding of the value this feeds.  One MUFU (ex2) + ~13 FMA-pipe
// instructions per element - erff costs ~30, and two MUFUs made the fc1 epilogue MUFU-bound.
//
// The array forms evaluate N elements stage by stage (every element's z, then every element's next polynomial term, ...):
// the N independent chains are then interleaved in the instruction stream.  Written element by element, ptxas kept
// each ~100-clock dependent chain whole in the register-lean epilogue warpgroup, and a GELU tile took ~12 k clocks.
// The arithmetic of each element is the same either way.
template <int N>
__device__ __forceinline__ void gelu_erf_n(float* x) {
    float z[N], q[N];
#pragma unroll
    for (int i = 0; i < N; ++i) { z[i] = fminf(fabsf(x[i]) * 0.70710678118654752f, 4.3f); q[i] = 1.04899843e-04f; }
    constexpr float kQ[6] = {-4.92790774e-04f, -2.22368206e-03f, 2.93586859e-02f, -1.48908889e-01f, -9.18342944e-01f,
                             -1.62791250e+00f};
#pragma unroll
    for (int t = 0; t < 6; ++t) {
#pragma unroll
        for (int i = 0; i < N; ++i) q[i] = fmaf(q[i], z[i], kQ[t]);
    }
#pragma unroll
    for (int i = 0; i < N; ++i) asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(q[i]) : "f"(q[i] * z[i]));
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = 0.5f * x[i] * (1.0f + copysignf(1.0f - q[i], x[i]));
}
__device__ __forceinline__ float gelu_erf(float x) {
    gelu_erf_n<1>(&x);
    return x;
}

// ELU (alpha = 1) in ~10 instructions (expm1f is ~25, in an epilogue that is issue-bound): the negative branch is
// 2^(x log2 e) - 1 with one MUFU (absolute error 2^-22) below -1/16, and the Taylor polynomial of degree 4 above it, where
// the subtraction would cancel (truncation < 8e-9, relative error ~1e-7 of a result that is then rounded to fp16).
// Stage by stage over N elements, as gelu_erf_n.
template <int N>
__device__ __forceinline__ void elu_ex2_n(float* x) {
    float e[N], t[N];
#pragma unroll
    for (int i = 0; i < N; ++i) asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e[i]) : "f"(fminf(x[i], 0.f) * 1.4426950408889634f));
#pragma unroll
    for (int i = 0; i < N; ++i) t[i] = x[i] * fmaf(x[i], fmaf(x[i], fmaf(x[i], 4.16666667e-2f, 1.66666667e-1f), 0.5f), 1.0f);
#pragma unroll
    for (int i = 0; i < N; ++i) x[i] = x[i] > 0.f ? x[i] : (x[i] > -0.0625f ? t[i] : e[i] - 1.0f);
}

__device__ __forceinline__ uint32_t hmax2_u32(uint32_t a, uint32_t b) {
    __half2 r = __hmax2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&b));
    return *reinterpret_cast<uint32_t*>(&r);
}

template <int N_TILE, int STAGES, int WMODE>
__global__ void __launch_bounds__(kConvGemmThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap map_x,
                 const __grid_constant__ CUtensorMap map_w,
                 const ConvGemmParams p)
{
    using namespace sm90;
    static_assert(N_TILE == 128, "one m64n128 accumulator per consumer warpgroup");
    static_assert(WMODE == 0 || WMODE == 1, "WMODE 0: fp16 weights, 1: fp16 hi/lo pair");
    static_assert(kClusterCtas == 2, "the work units below are M-tile pairs");
    constexpr bool SPLIT_W = WMODE == 1;
    constexpr uint32_t kStageBytes = conv_gemm_stage_bytes<N_TILE, WMODE>();
    constexpr int kBRows = (SPLIT_W ? 2 : 1) * N_TILE;              // rows of the packed weight tensor per N tile
    constexpr int kGroups = N_TILE / 32;                // epilogue: one row per lane, 32 columns (one 128-B segment) per group

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * kStageBytes);
    uint64_t* full = bars;
    uint64_t* empty = bars + STAGES;
    uint64_t* epi_full = bars + 2 * STAGES;                         // [kConsumers]: consumer c's half is in the tile
    uint64_t* epi_empty = bars + 2 * STAGES + kConsumers;           // [kConsumers]: the epilogue is done with it
    static_assert((2 * STAGES + 2 * kConsumers) * 8 <= 256, "barriers");
    uint8_t* epi = smem + STAGES * kStageBytes + 256;                // kConsumers x kEpiBytes, then 4 x kBiasBytes

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int ksteps = p.taps * p.cblks;
    const int n_chunks = (ksteps + kChunkSteps - 1) / kChunkSteps;
    const int chunk_len = (ksteps + n_chunks - 1) / n_chunks;       // balanced chunks
    const int m_tiles = p.img_groups * p.tiles_h * p.tiles_w;
    // work unit = (M-tile pair, N tile), N fastest; this CTA computes M tile 2 * pair + rank of each unit.  Each role reads
    // its cluster index and rank after its setmaxnreg: kept live across the role split, they were spilled.
    const int n_clusters = (int)gridDim.x / kClusterCtas;
    const int total_units = (m_tiles + 1) / 2 * p.n_tiles;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&map_x);
        tma_prefetch_desc(&map_w);
    }
    if (warp == 1 && lane == 0) {
        // empty[s]: one arrival per consumer warp of both CTAs (the partner's multicast writes into this stage too)
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kClusterCtas * kConsumers * 4); }
        // epi_full[c]: every thread of consumer c; epi_empty[c]: every thread of the two epilogue warps of half c
        for (int c = 0; c < kConsumers; ++c) { mbar_init(&epi_full[c], 128); mbar_init(&epi_empty[c], 64); }
        mbar_fence_init();
    }
    cluster_sync();                                   // both CTAs' barriers exist before any multicast or remote arrive

    if (warp < 4) {
        // ------------------------------------------------------------ TMA producer
        // hand the registers of this warpgroup to the two consumers, which hold 2 x 64 fp32 accumulators
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            const int rank = (int)cluster_ctarank();
            const int cluster = (int)cluster_index();
            constexpr int kHalfRows = kBRows / kClusterCtas;              // weight rows this rank loads per k-step
            uint8_t* const w_half = smem + kABytes + rank * kHalfRows * 128;
            int s = 0; uint32_t ph = 0;
            for (int unit = cluster; unit < total_units; unit += n_clusters) {
                const int nt = unit % p.n_tiles;
                const int m = min(2 * (unit / p.n_tiles) + rank, m_tiles - 1);   // the spare reads rank 0's rows
                const int w0 = (m % p.tiles_w) * p.box_w;
                const int h0 = ((m / p.tiles_w) % p.tiles_h) * p.box_h;
                const int n0 = (m / (p.tiles_w * p.tiles_h)) * p.box_n;
                for (int ks = 0; ks < ksteps; ++ks) {
                    const int tap = ks / p.cblks;
                    const int cb = ks - tap * p.cblks;
                    int dh = 0, dw = 0;
                    if (p.taps == 9) { dh = tap / 3 - 1; dw = tap % 3 - 1; }
                    mbar_wait(&empty[s], ph ^ 1);
                    uint8_t* st = smem + s * kStageBytes;
                    mbar_expect_tx(&full[s], kStageBytes);
                    tma_load_4d(st, &map_x, &full[s], cb * kBlockK, w0 + dw, h0 + dh, n0);
                    tma_load_2d_multicast(w_half + s * kStageBytes, &map_w, &full[s], ks * kBlockK,
                                          nt * kBRows + rank * kHalfRows, (1u << kClusterCtas) - 1);
                    if (++s == STAGES) { s = 0; ph ^= 1; }
                }
            }
        }
    } else if (warp < 4 + 4 * kConsumers) {
        // ------------------------------------------------------------ consumers: wgmma + chunk fold + fragment dump
        setmaxnreg_inc<kConsumerRegs>();
        const int cluster = (int)cluster_index();
        const int c = (warp >> 2) - 1;                    // consumer index: tile rows [64 c, 64 c + 64)
        const int wq = warp & 3;                          // warp within the warpgroup
        const uint32_t epi_base = smem_u32(epi) + c * kEpiBytes;
        int s = 0; uint32_t ph = 0, eph = 0;
        // a stage is free once the consumer warps of both CTAs have read it
        auto release = [&](int st_) {
            __syncwarp();
            if (lane == 0) {
#pragma unroll
                for (int cta = 0; cta < kClusterCtas; ++cta) mbar_arrive_cluster(&empty[st_], cta);
            }
        };

        for (int unit = cluster; unit < total_units; unit += n_clusters) {
            // ---- main loop: chunks of <= kChunkSteps k-steps into `acc`, summed into `sum` (round-to-nearest adds,
            // undoing the expected truncation shrink of each chunk)
            float sum[64], acc[64];
#pragma unroll
            for (int i = 0; i < 64; ++i) sum[i] = 0.f;
            for (int ks0 = 0; ks0 < ksteps; ks0 += chunk_len) {
                const int ks1 = min(ks0 + chunk_len, ksteps);
                // products accumulated per accumulator element: the truncation acts on the running sum, so the lo-part
                // wgmmas that share the accumulator (SPLIT_W) shrink it as much as the hi ones although their products
                // are ~2^-11 of them (tests/test_gpu_gemm.py::test_accumulation_is_unbiased: counting only K leaves
                // -5e-7 per 512-K chunk on H100).  All-zero lo parts (weights exact in fp16, p.lo_adds = 0) add exact
                // zeros, which do not truncate: counting them would over-correct by +5.4e-7 per chunk.
                const float unshrink = kAccumShrinkPerElement * (float)((ks1 - ks0) * kBlockK * (SPLIT_W && p.lo_adds ? 2 : 1));
                int prev_s = -1;
                for (int ks = ks0; ks < ks1; ++ks) {
                    mbar_wait(&full[s], ph);
                    const uint32_t a_addr = smem_u32(smem + s * kStageBytes);
                    const uint64_t a_desc = kmajor_sw128_desc(a_addr + c * 64 * 128);     // this consumer's 64 rows
                    const uint64_t b_desc = kmajor_sw128_desc(a_addr + kABytes);
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < kBlockK / 16; ++k) {
                        // +32 B along K inside the 128-B swizzle atom == +2 in the 16-B address field
                        wgmma_m64n128k16_f16<0, 0>(acc, a_desc + 2 * k, b_desc + 2 * k, (ks > ks0) || (k > 0));
                        if (SPLIT_W)                   // lo rows: N_TILE rows (x 128 B) further down the stage, same accumulator
                            wgmma_m64n128k16_f16<0, 0>(acc, a_desc + 2 * k, b_desc + 2 * k + (N_TILE * 128 / 16), 1);
                    }
                    wgmma_commit();
                    wgmma_wait<1>();                   // the previous k-step's wgmmas have retired: release its stage
                    if (prev_s >= 0) release(prev_s);
                    prev_s = s;
                    if (++s == STAGES) { s = 0; ph ^= 1; }
                }
                wgmma_wait<0>();
                fence_regs(acc);
                release(prev_s);
#pragma unroll
                for (int i = 0; i < 64; ++i) sum[i] += fmaf(acc[i], unshrink, acc[i]);
            }

            // ---- accumulator fragment -> this consumer's half of the fp32 tile [64 rows][128 cols] in shared memory,
            // 16-B chunks XOR-swizzled by row, once the epilogue has drained the previous tile's half; the arrive
            // releases the stores to it
            mbar_wait(&epi_empty[c], eph ^ 1);
            // element (row, col) = (fr + 8 i, 8 j + 2 (lane % 4) + e) sits in 16-B chunk (col / 4) ^ (row % 8) of its row;
            // with j = 4 jh + jl that is 8 jh + ((2 jl) ^ x), so four base registers and immediate offsets cover all 32
            const int fr = wq * 16 + (lane >> 2);
            const uint32_t x = ((lane & 3) >> 1) ^ (fr & 7);
            const uint32_t row_base = epi_base + fr * kEpiRowBytes + (lane & 1) * 8;
#pragma unroll
            for (int jl = 0; jl < 4; ++jl) {
                const uint32_t a = row_base + (((2 * jl) ^ x) << 4);
#pragma unroll
                for (int jh = 0; jh < 4; ++jh) {
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int j = 4 * jh + jl;
                        sts64(a + i * 8 * kEpiRowBytes + jh * 128, sum[4 * j + 2 * i], sum[4 * j + 2 * i + 1]);
                    }
                }
            }
            mbar_arrive(&epi_full[c]);
            eph ^= 1;
        }
    } else {
        // ------------------------------------------------------------ epilogue: one tile row per lane
        // every warp starts at the launch allocation of 65536 / 512 = 128 registers; setmaxnreg.dec may only lower it
        if constexpr (kEpiRegs > 65536 / kConvGemmThreads) setmaxnreg_inc<kEpiRegs>();
        else setmaxnreg_dec<kEpiRegs>();
        const int rank = (int)cluster_ctarank();
        const int cluster = (int)cluster_index();
        const int e = warp - 4 - 4 * kConsumers;         // epilogue warp 0..3
        const int c = e >> 1;                             // it drains consumer c's half ...
        const int rr = (e & 1) * 32 + lane;               // ... row rr of it
        const int r = c * 64 + rr;                        // row of the tile
        const int bw = p.box_w, bh = p.box_h;
        const int pw = r % bw;
        const int phh = (r / bw) % bh;
        const int pn = r / (bw * bh);
        // this warp's 32 rows of the tile; the 128-B segment of group g of each row doubles as its output staging once read
        const uint32_t wrows = smem_u32(epi) + c * kEpiBytes + (e & 1) * 32 * kEpiRowBytes;
        const uint32_t row_mine = wrows + lane * kEpiRowBytes;
        const uint32_t bias_s = smem_u32(epi) + kConsumers * kEpiBytes + e * kBiasBytes;
        const int sw = lane & 7;                          // == rr & 7 == r & 7: the swizzle of this lane's row
        const int cq = lane & 7, rq = lane >> 3;          // flush role: 16-B chunk cq of rows it*4 + rq
        uint32_t eph = 0;
        // plain row-major GEMM (1x1 "image", 128 rows per tile): no per-tile divisions
        const bool plain = p.tiles_w == 1 && p.tiles_h == 1 && bw == 1 && bh == 1;
        const bool f32_path = p.out_f32 != nullptr || p.resid != nullptr;
        // residual rows are read-modify-written here: pull the NEXT tile's rows into L2 while this one is stored,
        // so the loads do not pay HBM latency on the critical path
        auto prefetch_resid = [&](int nt_, int m_) {
            if (p.resid == nullptr || !plain) return;
            const int n_ = m_ * kTileM + r;
            if (n_ >= p.NB) return;
            const long long tok = p.resid_res ? window_row_to_token((long long)n_, p.resid_res, p.resid_shift) : (long long)n_;
            for (int cc = nt_ * N_TILE; cc < nt_ * N_TILE + N_TILE && cc < p.resid_C; cc += 32)
                asm volatile("prefetch.global.L2 [%0];" :: "l"(p.resid + tok * p.resid_C + cc));
        };
        if (cluster < total_units) prefetch_resid(cluster % p.n_tiles, 2 * (cluster / p.n_tiles) + rank);

        for (int unit = cluster; unit < total_units; unit += n_clusters) {
            const int nt = unit % p.n_tiles;
            const int m = 2 * (unit / p.n_tiles) + rank;       // == m_tiles on the spare: every row is >= NB
            if (unit + n_clusters < total_units)
                prefetch_resid((unit + n_clusters) % p.n_tiles, 2 * ((unit + n_clusters) / p.n_tiles) + rank);
            // the tile's bias into this warp's slice (broadcast reads below), before the wait
            __syncwarp();                                 // the previous tile's reads of the slice are done
            {
                const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + nt * N_TILE) + lane);
                sts128(bias_s + lane * 16, __float_as_uint(b.x), __float_as_uint(b.y), __float_as_uint(b.z), __float_as_uint(b.w));
            }
            __syncwarp();

            int w, h, n;
            if (plain) { w = 0; h = 0; n = m * kTileM + r; }
            else {
                w = (m % p.tiles_w) * bw + pw;
                h = ((m / p.tiles_w) % p.tiles_h) * bh + phh;
                n = (m / (p.tiles_w * p.tiles_h)) * p.box_n + pn;
            }
            const bool valid = n < p.NB;
            const int ch0 = nt * N_TILE;
            // Destination of this lane's row (element offsets, -1 = row beyond the batch).  Stores go through the
            // warp's rows of the tile (16-B chunks XOR-swizzled by row) so a warp writes whole 128-B lines of 4 rows
            // per instruction instead of 16 B into 32 different rows.
            long long out_off = -1, res_off = -1;
            if (valid && !p.pool) {
                out_off = (long long)((size_t(n) * p.H + h) * p.W + w) * p.ld_out;
                if (p.resid != nullptr)
                    res_off = (p.resid_res ? window_row_to_token((long long)n, p.resid_res, p.resid_shift) : (long long)n)
                              * p.resid_C;
            }

            mbar_wait(&epi_full[c], eph);
#pragma unroll 1
            for (int g = 0; g < kGroups; ++g) {
                float f[32];
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const uint4 u = lds128(row_mine + g * 128 + ((j ^ sw) << 4));
                    const uint4 b = lds128(bias_s + g * 128 + j * 16);
                    f[4 * j + 0] = __uint_as_float(u.x) + __uint_as_float(b.x);
                    f[4 * j + 1] = __uint_as_float(u.y) + __uint_as_float(b.y);
                    f[4 * j + 2] = __uint_as_float(u.z) + __uint_as_float(b.z);
                    f[4 * j + 3] = __uint_as_float(u.w) + __uint_as_float(b.w);
                }
                if (p.relu == 1) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j], 0.0f);
                } else if (p.relu == 2) {
#pragma unroll
                    for (int j = 0; j < 32; j += 8) gelu_erf_n<8>(f + j);
                } else if (p.relu == 3) {                           // ELU (alpha = 1): SEANet's activation
#pragma unroll
                    for (int j = 0; j < 32; j += 8) elu_ex2_n<8>(f + j);
                }

                if (!p.pool) {
                    if (f32_path) {
                        if (p.out != nullptr && out_off >= 0) {   // rare: both precisions; the fp16 copy direct, in 8-column pieces
                            uint4* dst = reinterpret_cast<uint4*>(p.out + out_off + ch0 + g * 32);
#pragma unroll
                            for (int j = 0; j < 4; ++j)          // n_valid is a multiple of 8: a partial last group
                                if (ch0 + g * 32 + 8 * j < p.n_valid)
                                    dst[j] = make_uint4(pack_half2(f[8 * j], f[8 * j + 1]), pack_half2(f[8 * j + 2], f[8 * j + 3]),
                                                        pack_half2(f[8 * j + 4], f[8 * j + 5]), pack_half2(f[8 * j + 6], f[8 * j + 7]));
                        }
                        // fp32 outputs: this group's 32 columns = one 128-B row segment per row, staged in place
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            sts128(row_mine + g * 128 + ((j ^ sw) << 4), __float_as_uint(f[4 * j]), __float_as_uint(f[4 * j + 1]),
                                   __float_as_uint(f[4 * j + 2]), __float_as_uint(f[4 * j + 3]));
                        __syncwarp();
                        const int col = ch0 + g * 32 + cq * 4;
#pragma unroll
                        for (int hf = 0; hf < 2; ++hf) {                   // 4 rows at a time: 4 loads in flight, then 4 stores
                            float4 v[4];
#pragma unroll
                            for (int it = 0; it < 4; ++it) {
                                const int x = (hf * 4 + it) * 4 + rq;
                                const uint4 u = lds128(wrows + x * kEpiRowBytes + g * 128 + ((cq ^ (x & 7)) << 4));
                                v[it] = make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
                            }
                            if (p.out_f32 != nullptr) {
#pragma unroll
                                for (int it = 0; it < 4; ++it) {
                                    const long long off = __shfl_sync(0xffffffffu, out_off, (hf * 4 + it) * 4 + rq);
                                    if (off >= 0 && col < p.n_valid) *reinterpret_cast<float4*>(p.out_f32 + off + col) = v[it];
                                }
                            }
                            if (p.resid != nullptr && ch0 + g * 32 < p.resid_C) {     // resid_C is a multiple of 32
                                long long offs[4];
                                float4 xv[4];
#pragma unroll
                                for (int it = 0; it < 4; ++it) {
                                    offs[it] = __shfl_sync(0xffffffffu, res_off, (hf * 4 + it) * 4 + rq);
                                    if (offs[it] >= 0) xv[it] = *reinterpret_cast<const float4*>(p.resid + offs[it] + col);
                                }
#pragma unroll
                                for (int it = 0; it < 4; ++it) {
                                    if (offs[it] >= 0) {
                                        const float4 a = v[it];
                                        xv[it].x += a.x; xv[it].y += a.y; xv[it].z += a.z; xv[it].w += a.w;
                                        *reinterpret_cast<float4*>(p.resid + offs[it] + col) = xv[it];
                                    }
                                }
                            }
                        }
                    } else if (p.out != nullptr) {
                        // fp16 output: groups g - 1 and g (64 columns) fill the 128-B segment of group g - 1, then flush
                        const int seg = (g & ~1) * 128;
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            sts128(row_mine + seg + ((((g & 1) * 4 + j) ^ sw) << 4),
                                   pack_half2(f[8 * j], f[8 * j + 1]), pack_half2(f[8 * j + 2], f[8 * j + 3]),
                                   pack_half2(f[8 * j + 4], f[8 * j + 5]), pack_half2(f[8 * j + 6], f[8 * j + 7]));
                        if (g & 1) {
                            __syncwarp();
                            const int col = ch0 + (g - 1) * 32 + cq * 8;
#pragma unroll
                            for (int it = 0; it < 8; ++it) {
                                const int x = it * 4 + rq;
                                const uint4 v = lds128(wrows + x * kEpiRowBytes + seg + ((cq ^ (x & 7)) << 4));
                                const long long off = __shfl_sync(0xffffffffu, out_off, x);
                                if (off >= 0 && col < p.n_valid) *reinterpret_cast<uint4*>(p.out + off + col) = v;
                            }
                        }
                    }
                } else {
                    uint32_t h2[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) h2[j] = pack_half2(f[2 * j], f[2 * j + 1]);
                    // 2x2 max-pool: partners are lane^1 (w) and lane^box_w (h), box_w in {8,16}
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        uint32_t o = __shfl_xor_sync(0xffffffffu, h2[j], 1);
                        h2[j] = hmax2_u32(h2[j], o);
                        o = __shfl_xor_sync(0xffffffffu, h2[j], bw);
                        h2[j] = hmax2_u32(h2[j], o);
                    }
                    // the four lanes of a 2x2 group now hold the same 32 channels; each stores 8
                    const int sub = (pw & 1) | ((phh & 1) << 1);
                    uint4 o;
                    o.x = sub == 0 ? h2[0] : sub == 1 ? h2[4] : sub == 2 ? h2[8]  : h2[12];
                    o.y = sub == 0 ? h2[1] : sub == 1 ? h2[5] : sub == 2 ? h2[9]  : h2[13];
                    o.z = sub == 0 ? h2[2] : sub == 1 ? h2[6] : sub == 2 ? h2[10] : h2[14];
                    o.w = sub == 0 ? h2[3] : sub == 1 ? h2[7] : sub == 2 ? h2[11] : h2[15];
                    if (valid) {
                        const size_t pix = (size_t(n) * (p.H >> 1) + (h >> 1)) * (p.W >> 1) + (w >> 1);
                        *reinterpret_cast<uint4*>(p.out + pix * p.Cout + ch0 + g * 32 + sub * 8) = o;
                    }
                }
            }
            mbar_arrive(&epi_empty[c]);                   // this lane's reads of the half are done
            eph ^= 1;
        }
    }
    cluster_sync();                                   // the partner's last arrivals on this CTA's barriers have landed
}

}  // namespace fad
