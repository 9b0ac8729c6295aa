// Encodec-24 kHz SEANet encoder (EncodecEmbModel, fadtk/model_loader.py:111-176: model.encoder(audio) ->
// [T/320, 128]) around the wgmma GEMM: every causal weight-normalised Conv1d is an im2col + GEMM (the
// pre-activation ELU is applied while gathering; reflect padding by index), residual blocks use the
// epilogue's fp32 read-modify-write, the 2-layer LSTM runs its input projections as one GEMM per layer and
// its recurrence as one small GEMM + cell kernel per time step.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace fad {

__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }

// channels = 2: the mono file duplicated to stereo, as encodec.utils.convert_audio does for the 48 kHz model
__global__ void __launch_bounds__(256)
pcm_to_f32_kernel(const int16_t* __restrict__ pcm, long long n, float* __restrict__ out, int channels = 1)
{
    for (long long i = blockIdx.x * 256LL + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const float v = (float)pcm[i] * (1.0f / 32768.0f);          // torchaudio.load normalisation (model_loader.py:168)
        if (channels == 1) out[i] = v;
        else { out[2 * i] = v; out[2 * i + 1] = v; }
    }
}

// GroupNorm(1, C) ("time_group_norm" of the 48 kHz model): statistics over all T x C values of one sample.
// stats[b] = {mean, rstd}; one block per sample.
__global__ void __launch_bounds__(1024)
groupnorm1_stats_kernel(const float* __restrict__ x, long long per_sample, float* __restrict__ stats)
{
    __shared__ double r1[1024], r2[1024];
    const float* xb = x + (size_t)blockIdx.x * per_sample;
    double s = 0.0, q = 0.0;
    for (long long i = threadIdx.x; i < per_sample; i += 1024) { const double v = xb[i]; s += v; q += v * v; }
    r1[threadIdx.x] = s; r2[threadIdx.x] = q;
    __syncthreads();
    for (int k = 512; k > 0; k >>= 1) {
        if (threadIdx.x < k) { r1[threadIdx.x] += r1[threadIdx.x + k]; r2[threadIdx.x] += r2[threadIdx.x + k]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double m = r1[0] / per_sample, var = r2[0] / per_sample - m * m;
        stats[2 * blockIdx.x] = (float)m; stats[2 * blockIdx.x + 1] = (float)(1.0 / sqrt(var + 1e-5));
    }
}
// x[b][t][c] = (x - mean_b) rstd_b gamma[c] + beta[c] (+ add[b][t][c]); optional fp16 copy
__global__ void __launch_bounds__(256)
groupnorm1_apply_kernel(float* __restrict__ x, const float* __restrict__ stats, const float* __restrict__ gamma,
                        const float* __restrict__ beta, const float* __restrict__ add, long long per_sample, int C, long long n,
                        __half* __restrict__ out16)
{
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < n; e += (long long)gridDim.x * 256) {
        const long long b = e / per_sample;
        const int c = (int)(e % C);
        float v = (x[e] - stats[2 * b]) * stats[2 * b + 1] * gamma[c] + beta[c];
        if (add != nullptr) v += add[e];
        x[e] = v;
        if (out16 != nullptr) out16[e] = __float2half_rn(v);
    }
}

// a[(b*T_out + t)][tap*C + c] = act(x[b][t*stride + tap - pad_left][c]).  Encodec's causal SConv1d pads
// pad_left = k - stride samples on the left and completes the last window on the right, both by reflection;
// a "valid" convolution (wav2vec2 feature encoder) passes pad_left = 0 and never leaves the signal.
// Encodec's pad1d reflects an input no longer than its padding (T_in <= max(pad_left, pad_right)) as if it had
// been extended with zeros to max_pad + 1 samples: the reflection runs over that length and taps past T_in read 0.
// kShort selects that case (enc_im2col decides per launch), so the loop of every longer input stays as it was.
// x: fp32 [B][T_in][C]; a: fp16 [B*T_out][Kpad] (columns >= k*C are zero).  One thread per 8 columns.
template <bool kShort>
__global__ void __launch_bounds__(256)
encodec_im2col_kernel(const float* __restrict__ x, int T_in, int C, int k, int stride, int pad_left, int elu, int T_out, int Kpad,
                      long long n_rows, __half* __restrict__ a)
{
    const int vecs = Kpad / 8, KC = k * C;
    int L = T_in;                                                   // length the reflection runs over
    if (kShort) {
        const int pad_right = (T_out - 1) * stride + k - pad_left - T_in;
        L = (pad_left > pad_right ? pad_left : pad_right) + 1;
    }
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < n_rows * vecs; e += (long long)gridDim.x * 256) {
        const long long row = e / vecs;
        const int col0 = (int)(e - row * vecs) * 8;
        const long long b = row / T_out;
        const int t = (int)(row - b * T_out);
        const float* xb = x + b * (long long)T_in * C;
        float v[8];
        if ((C & 7) == 0 && col0 + 8 <= KC) {                       // 8 channels of one tap: two float4 loads
            const int tap = col0 / C, c = col0 - tap * C;
            int i = t * stride + tap - pad_left;
            if (i < 0) i = -i;
            if (i >= L) i = 2 * (L - 1) - i;
            if (!kShort || i < T_in) {
                const float4 p = *reinterpret_cast<const float4*>(xb + (long long)i * C + c);
                const float4 q = *reinterpret_cast<const float4*>(xb + (long long)i * C + c + 4);
                v[0] = p.x; v[1] = p.y; v[2] = p.z; v[3] = p.w; v[4] = q.x; v[5] = q.y; v[6] = q.z; v[7] = q.w;
            } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] = 0.f;
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int col = col0 + j;
                float val = 0.f;
                if (col < KC) {
                    const int tap = col / C, c = col - tap * C;
                    int i = t * stride + tap - pad_left;
                    if (i < 0) i = -i;
                    if (i >= L) i = 2 * (L - 1) - i;
                    if (!kShort || i < T_in) val = xb[(long long)i * C + c];
                }
                v[j] = val;
            }
        }
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float p0 = v[2 * j], p1 = v[2 * j + 1];
            if (elu) {                                              // ELU(0) = 0: the zero padding columns stay zero
                p0 = elu1(p0); p1 = elu1(p1);
            }
            const __half2 hh = __floats2half2_rn(p0, p1);
            o[j] = *reinterpret_cast<const uint32_t*>(&hh);
        }
        *reinterpret_cast<uint4*>(a + row * Kpad + col0) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// One LSTM time step for G sequences (PyTorch gate order i, f, g, o):
//   gates = gx[b][t] (input projection + both biases) + rec[b] (h_{t-1} W_hh^T; absent at t = 0)
//   c = sigmoid(f) c + sigmoid(i) tanh(g);  h = sigmoid(o) tanh(c)
// h is handed to the next step's GEMM as an fp16 hi/lo pair [G][2H] (22 bits), y[b][t] = h (+ skip[b][t]).
__global__ void __launch_bounds__(256)
lstm_cell_kernel(const float* __restrict__ gx, const float* __restrict__ rec, int t, int T, int H, long long G,
                 float* __restrict__ c, __half* __restrict__ h16, float* __restrict__ y, const float* __restrict__ skip)
{
    for (long long e = blockIdx.x * 256LL + threadIdx.x; e < G * H; e += (long long)gridDim.x * 256) {
        const long long b = e / H;
        const int j = (int)(e - b * H);
        const float* g0 = gx + (b * T + t) * 4LL * H;
        float gi = g0[j], gf = g0[H + j], gg = g0[2 * H + j], go = g0[3 * H + j];
        if (rec != nullptr) {
            const float* r = rec + b * 4LL * H;
            gi += r[j]; gf += r[H + j]; gg += r[2 * H + j]; go += r[3 * H + j];
        }
        const float si = 1.0f / (1.0f + expf(-gi)), sf = 1.0f / (1.0f + expf(-gf)), so = 1.0f / (1.0f + expf(-go));
        const float cn = sf * (t == 0 ? 0.f : c[e]) + si * tanhf(gg);
        const float hn = so * tanhf(cn);
        c[e] = cn;
        const __half hh = __float2half_rn(hn);
        h16[b * 2 * H + j] = hh;
        h16[b * 2 * H + H + j] = __float2half_rn(hn - __half2float(hh));
        const long long yo = (b * T + t) * (long long)H + j;
        y[yo] = hn + (skip != nullptr ? skip[yo] : 0.f);
    }
}

}  // namespace fad
