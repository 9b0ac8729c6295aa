// wav2vec 2.0 / HuBERT / MERT style encoders (W2V2Model, HuBERTModel, MERTModel of fadtk/model_loader.py:
// processor normalisation -> 7-layer conv feature encoder -> feature projection -> grouped positional conv ->
// post-LN transformer layers -> hidden_states[layer]).  Convs and Linears run on the wgmma GEMM
// (operands read in place through overlapping-row tensor maps), attention on whisper_flash_attention_kernel, LayerNorm on clap_ln_kernel;
// this file adds the pieces those do not cover.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace fad {

// Wav2Vec2FeatureExtractor(do_normalize=True): x = (x - mean) / sqrt(var + 1e-7) per clip.  One block per clip.
__global__ void __launch_bounds__(1024)
w2v_normalize_kernel(const int16_t* __restrict__ pcm, int L, float* __restrict__ out)
{
    __shared__ double r1[1024], r2[1024];
    const int16_t* src = pcm + (size_t)blockIdx.x * L;
    double s = 0.0, q = 0.0;
    for (int i = threadIdx.x; i < L; i += 1024) { const double v = (double)src[i] * (1.0 / 32768.0); s += v; q += v * v; }
    r1[threadIdx.x] = s; r2[threadIdx.x] = q;
    __syncthreads();
    for (int k = 512; k > 0; k >>= 1) {
        if (threadIdx.x < k) { r1[threadIdx.x] += r1[threadIdx.x + k]; r2[threadIdx.x] += r2[threadIdx.x + k]; }
        __syncthreads();
    }
    const double mean = r1[0] / L, var = r2[0] / L - mean * mean;
    const float m = (float)mean, inv = (float)(1.0 / sqrt(var + 1e-7));
    float* dst = out + (size_t)blockIdx.x * L;
    for (int i = threadIdx.x; i < L; i += 1024) dst[i] = ((float)src[i] * (1.0f / 32768.0f) - m) * inv;
}

// ---- conv 0 of the group-norm feature encoder, fused: Conv1d(1, 512, k = 10, stride 5) -> GroupNorm(512, 512)
// -> GELU, written once as fp16.  GroupNorm's per-(clip, channel) statistics over time are linear / quadratic
// forms of the clip's window moments: with y[t][c] = sum_j w[c][j] x[5t + j] + b[c],
//   mean_t y = w[c] . m + b[c],   var_t y = w[c]^T (R - m m^T) w[c],
//   m[j] = mean_t x[5t + j],  R[j][j'] = mean_t x[5t + j] x[5t + j'],
// so the fp32 [T][512] conv output never exists in HBM (it was written once and read three times before).
// Moments and the 10 x 10 forms are evaluated in fp64.

// Per-(clip, slice) window moments, in fixed order so that the GroupNorm coefficients are reproducible bit for bit:
// part[b][s][0..9] = sum_t x[5t + j],  part[b][s][10 + j(j+1)/2 + j'] = sum_t x[5t + j] x[5t + j']  (j' <= j)
// over the frames t of slice s.  grid (kW2vMomSlices, B).
constexpr int kW2vMomSlices = 32;
__global__ void __launch_bounds__(256)
w2v_conv0_moments_kernel(const float* __restrict__ xn, int L, int T1, double* __restrict__ part /*[B][kW2vMomSlices][65]*/)
{
    __shared__ double red[8][65];
    const float* x = xn + (size_t)blockIdx.y * L;
    double a[65];
#pragma unroll
    for (int i = 0; i < 65; ++i) a[i] = 0.0;
    for (int t = blockIdx.x * 256 + threadIdx.x; t < T1; t += gridDim.x * 256) {
        double v[10];
#pragma unroll
        for (int j = 0; j < 10; ++j) v[j] = (double)x[5 * t + j];
#pragma unroll
        for (int j = 0; j < 10; ++j) {
            a[j] += v[j];
#pragma unroll
            for (int k = 0; k <= j; ++k) a[10 + j * (j + 1) / 2 + k] = fma(v[j], v[k], a[10 + j * (j + 1) / 2 + k]);
        }
    }
#pragma unroll
    for (int i = 0; i < 65; ++i) {
        double r = a[i];
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][i] = r;
    }
    __syncthreads();
    if (threadIdx.x < 65) {
        double r = 0.0;
        for (int w = 0; w < 8; ++w) r += red[w][threadIdx.x];
        part[((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 65 + threadIdx.x] = r;
    }
}

// coef[b][c] = (scale, shift) with GroupNorm(y)*gamma + beta = conv_nobias(x) * scale + shift.  One thread per (b, c).
__global__ void __launch_bounds__(256)
w2v_conv0_coef_kernel(const double* __restrict__ part /*[B][kW2vMomSlices][65]*/, const float* __restrict__ w /*[512][10]*/, const float* __restrict__ bias,
                      const float* __restrict__ gamma, const float* __restrict__ beta, int T1, int n /* B*512 */, float2* __restrict__ coef)
{
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const int b = i >> 9, c = i & 511;
    const double* p = part + (size_t)b * kW2vMomSlices * 65;
    auto a = [p](int k) {                            // moment k of the clip: its slices summed in slice order
        double r = p[k];
        for (int s = 1; s < kW2vMomSlices; ++s) r += p[s * 65 + k];
        return r;
    };
    const double inv = 1.0 / (double)T1;
    double wv[10], m[10];
    for (int j = 0; j < 10; ++j) { wv[j] = (double)w[c * 10 + j]; m[j] = a(j) * inv; }
    double mean = 0.0, var = 0.0;
    for (int j = 0; j < 10; ++j) {
        mean += wv[j] * m[j];
        for (int k = 0; k <= j; ++k) {
            const double cov = a(10 + j * (j + 1) / 2 + k) * inv - m[j] * m[k];
            var += (k == j ? 1.0 : 2.0) * wv[j] * wv[k] * cov;
        }
    }
    const double scale = (double)gamma[c] / sqrt(var + 1e-5);
    // y = conv + bias, mean_y = mean + bias: (y - mean_y) * scale + beta = conv * scale + (beta - mean * scale)
    (void)bias;
    coef[i] = make_float2((float)scale, (float)((double)beta[c] - mean * scale));
}

// out[b][t][c] = fp16(GELU(conv(x)[t][c] * scale + shift)) for t < T1, zeros for T1 <= t < P1 (row pitch P1 per clip,
// chosen so that the next layers can read their sliding windows as strided GEMM rows).
// grid (ceil(P1 / 128), B), 256 threads = 2 channels each.
__global__ void __launch_bounds__(256)
w2v_conv0_apply_kernel(const float* __restrict__ xn, int L, int T1, int P1, const float* __restrict__ w /*[512][10]*/,
                       const float2* __restrict__ coef /*[B][512]*/, __half* __restrict__ out)
{
    constexpr int TT = 128;
    __shared__ float xs[5 * TT + 8];
    const int b = blockIdx.y, t0 = blockIdx.x * TT;
    const float* x = xn + (size_t)b * L;
    for (int i = threadIdx.x; i < 5 * TT + 5; i += 256) { const int g = 5 * t0 + i; xs[i] = g < L ? x[g] : 0.f; }
    const int c = 2 * threadIdx.x;
    float w0[10], w1[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) { w0[j] = w[c * 10 + j]; w1[j] = w[c * 10 + 10 + j]; }
    const float2 k0 = coef[(size_t)b * 512 + c], k1 = coef[(size_t)b * 512 + c + 1];
    __syncthreads();
    __half2* o = reinterpret_cast<__half2*>(out + ((size_t)b * P1 + t0) * 512 + c);
    const int t_end = min(TT, P1 - t0);
    for (int t = 0; t < t_end; ++t) {
        float y0 = 0.f, y1 = 0.f;
        if (t0 + t < T1) {
#pragma unroll
            for (int j = 0; j < 10; ++j) { const float v = xs[5 * t + j]; y0 = fmaf(w0[j], v, y0); y1 = fmaf(w1[j], v, y1); }
            y0 = gelu_erf(fmaf(y0, k0.x, k0.y));
            y1 = gelu_erf(fmaf(y1, k1.x, k1.y));
        }
        o[(size_t)t * 256] = __floats2half2_rn(y0, y1);
    }
}

// Operand layout of the grouped positional convolution (k = 128, padding 64, 16 groups of cg channels; the
// even kernel's extra last output is dropped, Wav2Vec2SamePadLayer): per group a zero-padded fp16 sequence
//   a[g][b*Pp + p][ci] = h[b][p - 64][g*cg + ci]   (0 outside the clip),  Pp = T + 128,
// so that output (b, t) of group g is the contiguous run of 128*cg values starting at row b*Pp + t: a GEMM
// operand with row stride cg (overlapping rows) - no im2col copy.  Rows t >= T of every clip are dead.
// slab = rows per group (B*Pp + 128: the last dead rows read past the last clip).  8 channels per thread.
__global__ void __launch_bounds__(256)
w2v_posconv_layout_kernel(const float* __restrict__ h, int T, int d, int cg, int Pp, long long B, long long slab,
                          __half* __restrict__ a)
{
    const int per_row = cg / 8;
    const long long per_group = slab * per_row;
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < 16 * per_group; e += (long long)gridDim.x * 256) {
        const int g = (int)(e / per_group);
        const long long q = e - g * per_group;
        const long long row = q / per_row;
        const int ci = (int)(q - row * per_row) * 8;
        const long long b = row / Pp;
        const int t = (int)(row - b * Pp) - 64;
        uint4 o = make_uint4(0, 0, 0, 0);
        if (b < B && t >= 0 && t < T) {
            const float* src = h + ((b * T + t) * (long long)d + g * cg + ci);
            const float4 p = *reinterpret_cast<const float4*>(src), r = *reinterpret_cast<const float4*>(src + 4);
            const __half2 h0 = __floats2half2_rn(p.x, p.y), h1 = __floats2half2_rn(p.z, p.w);
            const __half2 h2 = __floats2half2_rn(r.x, r.y), h3 = __floats2half2_rn(r.z, r.w);
            o = make_uint4(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1),
                           *reinterpret_cast<const uint32_t*>(&h2), *reinterpret_cast<const uint32_t*>(&h3));
        }
        *reinterpret_cast<uint4*>(a + (g * slab + row) * cg + ci) = o;
    }
}

// out[b*T + t][col0 + c] = h[b*T + t][col0 + c] + y[b*Pp + t][c],  c < cg   (hidden + GELU(pos_conv(hidden)), one group)
__global__ void __launch_bounds__(256)
w2v_add_cols_kernel(const float* __restrict__ h, const float* __restrict__ y, long long n_rows, int T, int Pp, int d, int col0,
                    int cg, float* __restrict__ out)
{
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < n_rows * cg; e += (long long)gridDim.x * 256) {
        const long long row = e / cg;
        const int c = (int)(e - row * cg);
        const long long b = row / T;
        out[row * d + col0 + c] = h[row * d + col0 + c] + y[(b * Pp + (row - b * T)) * cg + c];
    }
}

// WavLM gated relative position bias (modeling_wavlm.WavLMAttention.forward steps 1-3): per (row, head)
//   p = W_g x_head + b_g (8 values);  a = sigmoid(p0+p1+p2+p3), b = sigmoid(p4+..+p7);  gate = a (b const_h - 1) + 2
// x: fp32 [rows][d] (the attention input), gate: [rows][heads].  One thread per (row, head).
__global__ void __launch_bounds__(256)
wavlm_gate_kernel(const float* __restrict__ x, const float* __restrict__ w /*[8][64]*/, const float* __restrict__ b /*[8]*/,
                  const float* __restrict__ cst /*[heads]*/, long long n_rows, int heads, int d, float* __restrict__ gate)
{
    __shared__ float ws[8 * 64 + 8];
    for (int i = threadIdx.x; i < 8 * 64 + 8; i += 256) ws[i] = i < 512 ? w[i] : b[i - 512];
    __syncthreads();
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < n_rows * heads; e += (long long)gridDim.x * 256) {
        const long long row = e / heads;
        const int hh = (int)(e - row * heads);
        const float* xr = x + row * d + hh * 64;
        float p[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) p[j] = ws[512 + j];
        for (int k = 0; k < 64; ++k) {
            const float xv = xr[k];
#pragma unroll
            for (int j = 0; j < 8; ++j) p[j] = fmaf(ws[j * 64 + k], xv, p[j]);
        }
        const float a = 1.0f / (1.0f + expf(-(p[0] + p[1] + p[2] + p[3])));
        const float bb = 1.0f / (1.0f + expf(-(p[4] + p[5] + p[6] + p[7])));
        gate[e] = a * (bb * cst[hh] - 1.0f) + 2.0f;
    }
}

__global__ void __launch_bounds__(256)
f32_to_f16_kernel(const float* __restrict__ x, long long n, __half* __restrict__ out)
{
    for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) out[i] = __float2half_rn(x[i]);
}

}  // namespace fad
