// Whisper (openai/whisper-{tiny..large}) as the reference uses it for embeddings
// (fadtk/model_loader.py:636-672): WhisperFeatureExtractor log-mel of the clip padded to 30 s ->
// WhisperModel(input_features, decoder_input_ids = [[sot, sot]]).last_hidden_state -> [2, d_model].
// The Linear / Conv1d layers run on the wgmma GEMM (conv_gemm.cuh, split fp16 weights); this file holds
// the CUDA-core / warp-MMA kernels around them:
//   whisper_logmel_kernel      |STFT_400|^2 (centre, reflect), 80 Slaney mel bands, log10, per-clip max
//   whisper_finish_im2col1     max(x, clipmax - 8), (x + 4) / 4, fp16, 3-tap im2col rows for conv1
//   whisper_im2col2            3-tap stride-2 im2col rows of conv1's output for conv2
//   whisper_pos_fill           residual stream <- positional embedding (conv2's GEMM then adds GELU(conv2))
//   whisper_flash_attention    encoder self-attention, 1500 x 1500 x 64 per head, mma.sync m16n8k16, online softmax
//   whisper_dec_self_attention 2 decoder tokens, causal
//   whisper_cross_attention    2 decoder queries against the 1500 encoder positions
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "clap.cuh"   // mma_m16n8k16, pack_h2

namespace fad {

constexpr int kWhFrames = 3000, kWhMel = 80, kWhFft = 400, kWhHop = 160, kWhBins = 201, kWhSamples = 480000;
constexpr int kWhMelTaps = 32;          // widest Slaney band at n_fft = 400 spans < 32 bins
constexpr int kWhFrameGroup = 8;        // frames per block
constexpr int kWhSeq = 1500;            // encoder positions

struct WhisperFrontTables {
    const float* cs;          // [400][2] cos, sin of 2 pi n / 400
    const float* hann;        // [400] periodic Hann
    const float* mel_w;       // [80][kWhMelTaps]
    const int* mel_start;     // [80]
    const int* mel_count;     // [80]
};

__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
    if (v >= 0.f) atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
    else atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// grid (3000 / 8, clips); block 256.  raw: [clips][3000][80] log10 mel; clip_max: [clips] (init -inf).
__global__ void __launch_bounds__(256)
whisper_logmel_kernel(const int16_t* __restrict__ pcm, const long long* __restrict__ clip_start,
                      const int* __restrict__ clip_len, WhisperFrontTables tab,
                      float* __restrict__ raw, float* __restrict__ clip_max)
{
    __shared__ float xw[kWhFrameGroup][kWhFft];
    __shared__ float2 cs[kWhFft];
    __shared__ float pw[kWhFrameGroup][kWhBins + 3];
    const int clip = blockIdx.y, f0 = blockIdx.x * kWhFrameGroup;
    const int len = min(clip_len[clip], kWhSamples);               // longer clips are truncated to 30 s
    float* dst = raw + ((size_t)clip * kWhFrames + f0) * kWhMel;
    // frames whose 400 samples all lie in the zero padding: mel = floor -> log10(1e-10) = -10
    if (f0 * kWhHop - kWhFft / 2 >= len && (f0 + kWhFrameGroup) * kWhHop + kWhFft / 2 < kWhSamples) {
        for (int i = threadIdx.x; i < kWhFrameGroup * kWhMel; i += 256) dst[i] = -10.0f;
        if (threadIdx.x == 0) atomic_max_float(clip_max + clip, -10.0f);
        return;
    }
    const int16_t* src = pcm + clip_start[clip];
    for (int i = threadIdx.x; i < kWhFft; i += 256) cs[i] = make_float2(tab.cs[2 * i], tab.cs[2 * i + 1]);
    for (int i = threadIdx.x; i < kWhFrameGroup * kWhFft; i += 256) {
        const int f = i / kWhFft, n = i - f * kWhFft;
        int s = (f0 + f) * kWhHop - kWhFft / 2 + n;                 // centre = True
        if (s < 0) s = -s;                                          // reflect padding of the 30-s buffer
        if (s >= kWhSamples) s = 2 * (kWhSamples - 1) - s;
        xw[f][n] = s < len ? (float)src[s] * (1.0f / 32768.0f) * tab.hann[n] : 0.0f;
    }
    __syncthreads();
    const int k = threadIdx.x;
    if (k < kWhBins) {
        float re[kWhFrameGroup], im[kWhFrameGroup];
#pragma unroll
        for (int f = 0; f < kWhFrameGroup; ++f) { re[f] = 0.f; im[f] = 0.f; }
        int idx = 0;
        for (int n = 0; n < kWhFft; ++n) {
            const float2 w = cs[idx];
#pragma unroll
            for (int f = 0; f < kWhFrameGroup; ++f) { const float x = xw[f][n]; re[f] = fmaf(x, w.x, re[f]); im[f] = fmaf(x, w.y, im[f]); }
            idx += k; if (idx >= kWhFft) idx -= kWhFft;
        }
#pragma unroll
        for (int f = 0; f < kWhFrameGroup; ++f) pw[f][k] = re[f] * re[f] + im[f] * im[f];
    }
    __syncthreads();
    float mx = -3.0e38f;
    for (int i = threadIdx.x; i < kWhFrameGroup * kWhMel; i += 256) {
        const int f = i / kWhMel, b = i - f * kWhMel;
        const int st = tab.mel_start[b], cnt = tab.mel_count[b];
        float acc = 0.f;
        for (int j = 0; j < cnt; ++j) acc = fmaf(pw[f][st + j], tab.mel_w[b * kWhMelTaps + j], acc);
        const float v = log10f(fmaxf(acc, 1e-10f));
        dst[i] = v;
        mx = fmaxf(mx, v);
    }
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0 && mx > -1.0e38f) atomic_max_float(clip_max + clip, mx);
}

// a1: fp16 [clips*3000][384] = im2col of the normalised log-mel for Conv1d(80 -> d, k = 3, pad = 1):
// column tap*128 + c holds y[t + tap - 1][c] (c < 80), zero elsewhere.
__global__ void __launch_bounds__(256)
whisper_finish_im2col1_kernel(const float* __restrict__ raw, const float* __restrict__ clip_max, long long n_rows,
                              __half* __restrict__ a1)
{
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < n_rows * 384; e += (long long)gridDim.x * 256) {
        const long long row = e / 384;
        const int col = (int)(e - row * 384);
        const int tap = col >> 7, c = col & 127;
        const long long clip = row / kWhFrames;
        const int t = (int)(row - clip * kWhFrames) + tap - 1;
        float y = 0.f;
        if (c < kWhMel && t >= 0 && t < kWhFrames) {
            const float x = fmaxf(raw[(clip * kWhFrames + t) * kWhMel + c], clip_max[clip] - 8.0f);
            y = (x + 4.0f) * 0.25f;
        }
        a1[e] = __float2half_rn(y);
    }
}

// a2: fp16 [clips*1500][3*d]: column tap*d + c = conv1_out[clip][2 t + tap - 1][c] (Conv1d k = 3, stride 2, pad 1)
__global__ void __launch_bounds__(256)
whisper_im2col2_kernel(const __half* __restrict__ h1 /*[clips*3000][d]*/, long long n_rows, int d, __half* __restrict__ a2)
{
    const int vec_per_row = 3 * d / 8;
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < n_rows * vec_per_row; e += (long long)gridDim.x * 256) {
        const long long row = e / vec_per_row;
        const int v = (int)(e - row * vec_per_row);
        const int col = v * 8, tap = col / d, c = col - tap * d;
        const long long clip = row / kWhSeq;
        const int t = 2 * (int)(row - clip * kWhSeq) + tap - 1;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (t >= 0 && t < kWhFrames) val = *reinterpret_cast<const uint4*>(h1 + ((clip * kWhFrames + t) * d + c));
        *reinterpret_cast<uint4*>(a2 + row * 3 * d + col) = val;
    }
}

// x[clip][t][:] = pos[t][:]   (fp32)
__global__ void __launch_bounds__(256)
whisper_pos_fill_kernel(const float* __restrict__ pos /*[rows_per_clip][d]*/, long long n_clips, int rows_per_clip, int d,
                        float* __restrict__ x)
{
    const long long per = (long long)rows_per_clip * d / 4;
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < n_clips * per; e += (long long)gridDim.x * 256)
        reinterpret_cast<float4*>(x)[e] = reinterpret_cast<const float4*>(pos)[e % per];
}

// Encoder self-attention.  qkv: fp16 [clips*S][3 d] (q | k | v, head h at h*64); out: fp16 [clips*S][d].
// grid (ceil(S / 64), heads, clips), 128 threads: each warp owns 16 query rows; K/V tiles of 64 keys are
// double-buffered with cp.async; S = Q K^T and O += P V on mma.sync m16n8k16 with an online softmax
// (scores scaled by 1/8 = head_dim^-0.5 as WhisperAttention does).
constexpr int kFaStride = 72;           // halves per smem row (64 used): conflict-free fragment loads / ldmatrix
__global__ void __launch_bounds__(128)
whisper_flash_attention_kernel(const __half* __restrict__ qkv, int S, int d, __half* __restrict__ out,
                               const float* __restrict__ relb = nullptr /* WavLM: [heads][2S-1] bias by key - query + S - 1 */,
                               const float* __restrict__ gate = nullptr /* WavLM: [clips*S][heads] per-query gate of that bias */)
{
    __shared__ __align__(16) __half q_s[64 * kFaStride];
    __shared__ __align__(16) __half kv_s[2][2][64 * kFaStride];     // [stage][k | v]
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int qb = blockIdx.x, h = blockIdx.y;
    const long long row0 = (long long)blockIdx.z * S;
    const int ld = 3 * d;
    const __half* base = qkv + row0 * ld + h * 64;
    auto load_tile = [&](__half* dst, const __half* src, int first_row) {          // 64 rows x 128 B
#pragma unroll
        for (int it = 0; it < 4; ++it) {
            const int i = it * 128 + threadIdx.x;
            const int r = i >> 3, v = i & 7;
            const int gr = first_row + r;
            const uint32_t daddr = (uint32_t)__cvta_generic_to_shared(dst + r * kFaStride + v * 8);
            const __half* s = src + (size_t)(gr < S ? gr : S - 1) * ld + v * 8;     // rows past S are masked later
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(daddr), "l"(s));
        }
    };
    const int n_tiles = (S + 63) / 64;
    load_tile(q_s, base, qb * 64);
    load_tile(kv_s[0][0], base + d, 0);
    load_tile(kv_s[0][1], base + 2 * d, 0);
    asm volatile("cp.async.commit_group;" ::: "memory");

    float o[8][4], m0 = -3.0e38f, m1 = -3.0e38f, l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int n = 0; n < 8; ++n) { o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f; }
    uint32_t qa[4][4];
    const float sc = 0.125f * 1.4426950408889634f;                  // head_dim^-0.5 and log2(e): softmax via exp2
    for (int tile = 0; tile < n_tiles; ++tile) {
        const int st = tile & 1;
        if (tile + 1 < n_tiles) {
            load_tile(kv_s[st ^ 1][0], base + d, (tile + 1) * 64);
            load_tile(kv_s[st ^ 1][1], base + 2 * d, (tile + 1) * 64);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncthreads();
        if (tile == 0) {
            const __half* qr = q_s + (warp * 16) * kFaStride;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                qa[ks][0] = *reinterpret_cast<const uint32_t*>(qr + g * kFaStride + ks * 16 + 2 * t);
                qa[ks][1] = *reinterpret_cast<const uint32_t*>(qr + (g + 8) * kFaStride + ks * 16 + 2 * t);
                qa[ks][2] = *reinterpret_cast<const uint32_t*>(qr + g * kFaStride + ks * 16 + 2 * t + 8);
                qa[ks][3] = *reinterpret_cast<const uint32_t*>(qr + (g + 8) * kFaStride + ks * 16 + 2 * t + 8);
            }
        }
        const __half* k_s = kv_s[st][0];
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
            const __half* kr = k_s + (j * 8 + g) * kFaStride + 2 * t;
#pragma unroll
            for (int ks = 0; ks < 4; ++ks)
                mma_m16n8k16(s[j], qa[ks][0], qa[ks][1], qa[ks][2], qa[ks][3],
                             *reinterpret_cast<const uint32_t*>(kr + ks * 16), *reinterpret_cast<const uint32_t*>(kr + ks * 16 + 8));
        }
        // scale (+ gated relative position bias), mask keys past S, running max
        const int key0 = tile * 64;
        float mx0 = m0, mx1 = m1;
        const int qr0 = qb * 64 + warp * 16 + g, qr1 = qr0 + 8;
        float g0 = 0.f, g1 = 0.f;
        const float* rb = nullptr;
        if (relb != nullptr) {
            rb = relb + (size_t)h * (2 * S - 1) + (S - 1);
            const int heads = gridDim.y;
            g0 = gate[(row0 + min(qr0, S - 1)) * heads + h];
            g1 = gate[(row0 + min(qr1, S - 1)) * heads + h];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int kc = key0 + j * 8 + 2 * t;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = kc + (e & 1);
                const bool valid = key < S;
                float v = s[j][e] * sc;
                if (rb != nullptr && valid) {
                    const int q_ = (e < 2) ? qr0 : qr1;
                    v = fmaf((e < 2 ? g0 : g1) * rb[key - min(q_, S - 1)], 1.4426950408889634f, v);
                }
                s[j][e] = valid ? v : -3.0e38f;
            }
            mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
            mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float a0 = exp2f(m0 - mx0), a1 = exp2f(m1 - mx1);
        m0 = mx0; m1 = mx1;
        float r0 = 0.f, r1 = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            s[j][0] = exp2f(s[j][0] - m0); s[j][1] = exp2f(s[j][1] - m0);
            s[j][2] = exp2f(s[j][2] - m1); s[j][3] = exp2f(s[j][3] - m1);
            r0 += s[j][0] + s[j][1]; r1 += s[j][2] + s[j][3];
        }
        l0 = l0 * a0 + r0; l1 = l1 * a1 + r1;                      // per-lane partial sums (reduced at the end)
#pragma unroll
        for (int n = 0; n < 8; ++n) { o[n][0] *= a0; o[n][1] *= a0; o[n][2] *= a1; o[n][3] *= a1; }
        const uint32_t v_ld = (uint32_t)__cvta_generic_to_shared(kv_s[st][1]) + ((lane & 15) * kFaStride + (lane >> 4) * 8) * 2;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint32_t p0 = pack_h2(s[2 * kk][0], s[2 * kk][1]), p1 = pack_h2(s[2 * kk][2], s[2 * kk][3]);
            const uint32_t p2 = pack_h2(s[2 * kk + 1][0], s[2 * kk + 1][1]), p3 = pack_h2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
            for (int np = 0; np < 4; ++np) {                        // two 8-dim n-tiles per ldmatrix.x4
                uint32_t b[4];
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(b[0]), "=r"(b[1]), "=r"(b[2]), "=r"(b[3]) : "r"(v_ld + (kk * 16 * kFaStride + np * 16) * 2));
                mma_m16n8k16(o[2 * np], p0, p1, p2, p3, b[0], b[1]);
                mma_m16n8k16(o[2 * np + 1], p0, p1, p2, p3, b[2], b[3]);
            }
        }
        __syncthreads();                                            // this stage may be overwritten by the next prefetch
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    const int q0 = qb * 64 + warp * 16 + g, q1 = q0 + 8;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
        if (q0 < S) *reinterpret_cast<uint32_t*>(out + (row0 + q0) * d + h * 64 + n * 8 + 2 * t) = pack_h2(o[n][0] * i0, o[n][1] * i0);
        if (q1 < S) *reinterpret_cast<uint32_t*>(out + (row0 + q1) * d + h * 64 + n * 8 + 2 * t) = pack_h2(o[n][2] * i1, o[n][3] * i1);
    }
}

// Decoder self-attention over the two start tokens (causal): token 0 sees itself, token 1 sees both.
// qkv: fp16 [clips*2][3 d]; out: fp16 [clips*2][d].  One warp per (clip, head); lane owns dims 2*lane, 2*lane+1.
__global__ void __launch_bounds__(128)
whisper_dec_self_attention_kernel(const __half* __restrict__ qkv, long long n_clips, int heads, int d, __half* __restrict__ out)
{
    const long long u = blockIdx.x * 4LL + (threadIdx.x >> 5);
    if (u >= n_clips * heads) return;
    const int lane = threadIdx.x & 31;
    const long long clip = u / heads;
    const int h = (int)(u - clip * heads);
    const __half* r0 = qkv + (clip * 2) * 3 * d + h * 64 + 2 * lane;
    const __half* r1 = r0 + 3 * d;
    const float2 q1 = __half22float2(*reinterpret_cast<const __half2*>(r1));
    const float2 k0 = __half22float2(*reinterpret_cast<const __half2*>(r0 + d));
    const float2 k1 = __half22float2(*reinterpret_cast<const __half2*>(r1 + d));
    const float2 v0 = __half22float2(*reinterpret_cast<const __half2*>(r0 + 2 * d));
    const float2 v1 = __half22float2(*reinterpret_cast<const __half2*>(r1 + 2 * d));
    float s0 = q1.x * k0.x + q1.y * k0.y, s1 = q1.x * k1.x + q1.y * k1.y;
    for (int o = 16; o > 0; o >>= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
    s0 *= 0.125f; s1 *= 0.125f;
    const float m = fmaxf(s0, s1), e0 = __expf(s0 - m), e1 = __expf(s1 - m), inv = 1.0f / (e0 + e1);
    __half* o0 = out + (clip * 2) * d + h * 64 + 2 * lane;
    *reinterpret_cast<__half2*>(o0) = __floats2half2_rn(v0.x, v0.y);
    *reinterpret_cast<__half2*>(o0 + d) = __floats2half2_rn((e0 * v0.x + e1 * v1.x) * inv, (e0 * v0.y + e1 * v1.y) * inv);
}

// Cross-attention: q fp16 [clips*2][d]; kv fp16 [clips*S][2 d] (k | v); out fp16 [clips*2][d].
// One block of 128 threads per (clip, head): scores of both queries against S keys, softmax, weighted V sum.
__global__ void __launch_bounds__(128)
whisper_cross_attention_kernel(const __half* __restrict__ q, const __half* __restrict__ kv, int S, int heads, int d,
                               __half* __restrict__ out)
{
    extern __shared__ float p_s[];                                  // [2][S]
    __shared__ float red[2][4];
    const int h = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long clip = blockIdx.y;
    const __half* kbase = kv + clip * S * 2 * d + h * 64;
    __shared__ float2 q_s[2][32];
    if (threadIdx.x < 64) {
        const int qi_ = threadIdx.x >> 5, i = threadIdx.x & 31;
        q_s[qi_][i] = __half22float2(*reinterpret_cast<const __half2*>(q + (clip * 2 + qi_) * d + h * 64 + 2 * i));
    }
    __syncthreads();
    float mx0 = -3.0e38f, mx1 = -3.0e38f;
    for (int k = threadIdx.x; k < S; k += 128) {
        const uint4* kr = reinterpret_cast<const uint4*>(kbase + (size_t)k * 2 * d);
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int v = 0; v < 8; ++v) {
            const uint4 w = kr[v];
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 kk = __half22float2(*reinterpret_cast<const __half2*>(&ws[e]));
                const float2 qa = q_s[0][v * 4 + e], qb = q_s[1][v * 4 + e];
                s0 = fmaf(qa.x, kk.x, fmaf(qa.y, kk.y, s0));
                s1 = fmaf(qb.x, kk.x, fmaf(qb.y, kk.y, s1));
            }
        }
        s0 *= 0.125f; s1 *= 0.125f;
        p_s[k] = s0; p_s[S + k] = s1;
        mx0 = fmaxf(mx0, s0); mx1 = fmaxf(mx1, s1);
    }
    auto block_reduce = [&](float v, int slot, bool is_max) -> float {
        for (int o = 16; o > 0; o >>= 1) { const float w = __shfl_xor_sync(0xffffffffu, v, o); v = is_max ? fmaxf(v, w) : v + w; }
        if (lane == 0) red[slot][warp] = v;
        __syncthreads();
        float r = red[slot][0];
        for (int i = 1; i < 4; ++i) r = is_max ? fmaxf(r, red[slot][i]) : r + red[slot][i];
        __syncthreads();
        return r;
    };
    mx0 = block_reduce(mx0, 0, true); mx1 = block_reduce(mx1, 1, true);
    float l0 = 0.f, l1 = 0.f;
    for (int k = threadIdx.x; k < S; k += 128) {
        const float e0 = __expf(p_s[k] - mx0), e1 = __expf(p_s[S + k] - mx1);
        p_s[k] = e0; p_s[S + k] = e1; l0 += e0; l1 += e1;
    }
    l0 = block_reduce(l0, 0, false); l1 = block_reduce(l1, 1, false);
    // thread (qi = tid / 64, dim = tid % 64)
    const int qi = threadIdx.x >> 6, dim = threadIdx.x & 63;
    const __half* vbase = kbase + d + dim;
    const float* pp = p_s + qi * S;
    float acc = 0.f;
    for (int k = 0; k < S; ++k) acc = fmaf(pp[k], __half2float(vbase[(size_t)k * 2 * d]), acc);
    out[(clip * 2 + qi) * d + h * 64 + dim] = __float2half_rn(acc / (qi ? l1 : l0));
}

}  // namespace fad
