// Encoder self-attention (head dim 64, no mask) on Hopper tensor cores: S = Q K^T and O = P V as wgmma tiles, the
// scores and the output accumulator in registers.
//
// Replaces the mma.sync flash kernel (whisper.cuh) on the Whisper / wav2vec 2.0 / HuBERT / MERT encoder paths - the
// reference's `WhisperModel(...)` / `AutoModel(...)` forwards (fadtk/model_loader.py:656-672, 254-288, 525-596) spend
// their attention time in torch SDPA; here one CTA owns a 128-query block of one (clip, head):
//
//   warpgroup 0     TMA producer (one elected lane): Q once, then K_j / V_j tiles (128 keys x 64 dims, 128-B swizzle)
//                   into a 2-stage ring.  The tensor map is 3-D [clips][S][3 d]: rows past S are zero-filled.
//   warpgroups 1-2  consumer c owns query rows [64 c, 64 c + 64): S_j = Q K_j^T (m64 n128 k16 x 4, both operands
//                   K-major in shared memory) into registers, online softmax in the exp2 domain on the accumulator
//                   fragment (a row lives in the four lanes of a quad), then O += P_j V_j (m64 n64 k16 x 8) with P
//                   as the register A operand - the S fragment of 16 keys IS the A fragment layout - and V as an
//                   MN-major B operand: the TMA tile [keys][dims] is that layout.
#pragma once
#include <cuda_bf16.h>
#include "sm90.cuh"

namespace fad {

constexpr int kAtThreads = 384;                                // producer warpgroup + two consumer warpgroups
constexpr uint32_t kAtTile = 128 * 128;                       // bytes of one 128-row x 64-col fp16 tile: 16 KiB
constexpr uint32_t kAtSmem = 1024 /*align slack*/ + kAtTile /*Q*/ + 2 * 2 * kAtTile /*K,V x 2 stages*/ + 256 /*barriers*/;

struct AttnParams {
    int S, d, heads;
    __half* out;             // [clips * S][d]
};

__global__ void __launch_bounds__(kAtThreads, 1)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap map_qkv, const AttnParams p)
{
    using namespace sm90;
    extern __shared__ uint8_t at_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* q_s = smem;
    uint8_t* kv_s = smem + kAtTile;                            // stage st: K at kv_s + st * 2 tiles, V one tile further
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 5 * kAtTile);
    uint64_t* q_full = bars;            // 1
    uint64_t* kv_full = bars + 1;       // 2
    uint64_t* kv_empty = bars + 3;      // 2

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qb = blockIdx.x, h = blockIdx.y, clip = blockIdx.z;
    const int n_blocks = (p.S + 127) / 128;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&map_qkv);
        mbar_init(q_full, 1);
        for (int i = 0; i < 2; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp < 4) {
        setmaxnreg_dec<40>();
        if (warp == 0 && elect_one()) {
            mbar_expect_tx(q_full, kAtTile);
            tma_load_3d(q_s, &map_qkv, q_full, h * 64, qb * 128, clip);
            for (int j = 0; j < n_blocks; ++j) {
                const int st = j & 1;
                mbar_wait(&kv_empty[st], ((j >> 1) & 1) ^ 1);
                mbar_expect_tx(&kv_full[st], 2 * kAtTile);
                uint8_t* kd = kv_s + st * 2 * kAtTile;
                tma_load_3d(kd, &map_qkv, &kv_full[st], p.d + h * 64, j * 128, clip);
                tma_load_3d(kd + kAtTile, &map_qkv, &kv_full[st], 2 * p.d + h * 64, j * 128, clip);
            }
        }
    } else {
        setmaxnreg_inc<232>();
        const int c = (warp >> 2) - 1;                         // consumer: query rows [64 c, 64 c + 64) of the block
        const int wq = warp & 3;
        const int t4 = lane & 3;
        const float sc = 0.125f * 1.4426950408889634f;         // head_dim^-0.5 and log2(e): softmax in the exp2 domain
        auto ex2 = [](float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; };
        float o[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] = 0.f;
        float m[2] = {-3.0e38f, -3.0e38f}, l[2] = {0.f, 0.f};  // rows r and r + 8 of this thread
        const uint64_t dq = kmajor_sw128_desc(smem_u32(q_s) + c * 64 * 128);
        mbar_wait(q_full, 0);
        for (int j = 0; j < n_blocks; ++j) {
            const int st = j & 1;
            const int valid = min(128, p.S - j * 128);          // keys of this block that exist
            mbar_wait(&kv_full[st], (j >> 1) & 1);
            const uint32_t kaddr = smem_u32(kv_s + st * 2 * kAtTile);
            const uint64_t dk = kmajor_sw128_desc(kaddr);
            float s[64];
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) wgmma_m64n128k16_f16<0, 0>(s, dq + 2 * k, dk + 2 * k, k > 0);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(s);
            if (valid < 128) {                                  // last block: zero-filled key rows take no weight
#pragma unroll
                for (int jj = 0; jj < 16; ++jj)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        if (8 * jj + 2 * t4 + e >= valid) { s[4 * jj + e] = -3.0e38f; s[4 * jj + 2 + e] = -3.0e38f; }
            }
            float alpha[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float r0 = s[2 * i], r1 = s[2 * i + 1];
#pragma unroll
                for (int jj = 1; jj < 16; ++jj) { r0 = fmaxf(r0, s[4 * jj + 2 * i]); r1 = fmaxf(r1, s[4 * jj + 2 * i + 1]); }
                float raw = fmaxf(r0, r1);
                raw = fmaxf(raw, __shfl_xor_sync(0xffffffffu, raw, 1));
                raw = fmaxf(raw, __shfl_xor_sync(0xffffffffu, raw, 2));
                const float mx = fmaxf(m[i], raw * sc);         // sc > 0: the maximum commutes with the scaling
                alpha[i] = ex2(m[i] - mx);
                m[i] = mx;
            }
            // P = fp16(exp2(s sc - m)), packed straight into the A fragments of the P V wgmmas; the row sum is taken over
            // the fp16 values the MMA reads (the weights of a row then sum to exactly 1)
            uint32_t pa[8][4];
            float rs[2] = {0.f, 0.f};
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {                   // q: (row half i = q & 1, column half = q >> 1)
                    const int i = q & 1;
                    const int base = 8 * kk + 4 * (q >> 1) + 2 * i;
                    const __half2 hh = __floats2half2_rn(ex2(fmaf(s[base], sc, -m[i])), ex2(fmaf(s[base + 1], sc, -m[i])));
                    pa[kk][q] = *reinterpret_cast<const uint32_t*>(&hh);
                    const float2 f = __half22float2(hh);
                    rs[i] += f.x + f.y;
                }
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) l[i] = l[i] * alpha[i] + rs[i];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
                o[4 * jj + 0] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
                o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
            }
            // V: [keys][dims] rows of 128 B = MN-major B (N = dims); 16 keys = two 8-row groups of 1024 B = +128 in the
            // 16-B address field
            const uint64_t dv = mnmajor_sw128_desc(kaddr + kAtTile, kAtTile, 1024);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) wgmma_m64n64k16_f16_rs(o, pa[kk], dv + 128 * kk, 1);
            wgmma_commit();
            wgmma_wait<0>();
            fence_regs(o);
            __syncwarp();
            if (lane == 0) mbar_arrive(&kv_empty[st]);
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {                           // the quad's partial row sums
            l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
            l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
        }
        const float inv[2] = {1.0f / l[0], 1.0f / l[1]};
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int q = qb * 128 + c * 64 + wq * 16 + (lane >> 2) + 8 * i;
            if (q < p.S) {
                __half* dst = p.out + ((size_t)clip * p.S + q) * p.d + h * 64 + 2 * t4;
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
                    *reinterpret_cast<__half2*>(dst + 8 * jj) = __floats2half2_rn(o[4 * jj + 2 * i] * inv[i], o[4 * jj + 2 * i + 1] * inv[i]);
            }
        }
    }
}

}  // namespace fad
