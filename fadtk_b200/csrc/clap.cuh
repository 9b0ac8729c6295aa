// CLAP-LAION audio branch (HTSAT-tiny Swin transformer) - the CUDA-core kernels around the
// wgmma GEMMs.  Replaces laion_clap / torchlibrosa behind CLAPLaionModel._get_embedding
// (fadtk/model_loader.py:389-411); architecture per SURVEY.md appendix B and the HF port of
// htsat.py (oracle/clap_oracle.py is pinned to it).
//
//   clap_logmel_kernel     int16 PCM window -> reference int16 round trip (:413-418) -> centre/reflect
//                          framing, Hann(1024), |rFFT_1024|^2, 64 Slaney mel bands, 10 log10(clamp),
//                          BatchNorm(eval) per mel bin -> fp32 [B, 1001, 64].  One warp per frame:
//                          512-point complex FFT = 16 (registers) x 32 (lanes, shuffles).
//   clap_patch_embed_kernel bicubic time resize 1001 -> 1024 (align_corners), fold into the 256x256
//                          "image", 4x4/4 conv 1 -> 96, LayerNorm -> fp32 residual stream [B,4096,96]
//   clap_ln_kernel         LayerNorm of the fp32 residual stream -> fp16 GEMM operand, rows emitted in
//                          (shifted-)window order, zero padded to the GEMM's K; merge mode gathers the
//                          2x2 neighbourhood (4C) for patch merging
//   clap_window_attention_kernel  softmax(q k^T / sqrt(24) + rel-pos bias (+ shift mask)) v per
//                          (window, head); fp32 math, one warp per unit
//   clap_residual_add_kernel      x[token] += y[row]  (row -> token is the inverse window map)
//   clap_head_kernel       final LayerNorm, token mean, 768->512 ReLU 512->512, L2 normalise -> fp16
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

#include "frontend.cuh"   // Cx, cmul, cadd, csub, mul_neg_i, shfl_xor_t
#include "conv_gemm.cuh"  // window_row_to_token

namespace fad {

constexpr int kClFft = 1024, kClHop = 480, kClMel = 64, kClChunk = 480000, kClFrames = 1001, kClBins = 513;
constexpr int kClMelTaps = 32;
constexpr int kClWarps = 8;

struct ClapFrontTables {
    const float* twiddle;    // [512][2] exp(-2 pi i k / 1024)
    const float* hann;       // [1024] periodic Hann
    const float* pcm_lut;    // [65536] reference int16 round trip: index = int16 + 32768
    const float* mel_w;      // [64][kClMelTaps]
    const int* mel_start;    // [64]
    const int* mel_count;    // [64]
    const float* bn_scale;   // [64] gamma / sqrt(var + eps)
    const float* bn_shift;   // [64] beta - mean * scale
};

__host__ __device__ constexpr size_t clap_logmel_smem_bytes() {
    return sizeof(float) * (size_t)(kClWarps * (2 * 512 + 516) + 2 * 512 + kClFft + kClMel * kClMelTaps + 2 * kClMel)
         + sizeof(int) * 2 * kClMel;
}

__device__ __forceinline__ void fft4(Cx<float>& a, Cx<float>& b, Cx<float>& c, Cx<float>& d) {
    const Cx<float> s0 = cadd(a, c), s1 = csub(a, c), s2 = cadd(b, d), s3 = mul_neg_i(csub(b, d));
    a = cadd(s0, s2); c = csub(s0, s2); b = cadd(s1, s3); d = csub(s1, s3);
}

// natural order in / out, forward transform; n = 4a + b, k = ka + 4 kb
__device__ __forceinline__ void fft16(Cx<float> (&x)[16]) {
    const float c1 = 0.92387953251128674f, s1 = 0.38268343236508977f, c2 = 0.70710678118654752f;
    // W16^m = (cos, -sin)(2 pi m / 16)
    const Cx<float> w1 = {c1, -s1}, w2 = {c2, -c2}, w3 = {s1, -c1}, w4 = {0.f, -1.f},
                    w6 = {-c2, -c2}, w9 = {-c1, s1};
#pragma unroll
    for (int b = 0; b < 4; ++b) fft4(x[b], x[4 + b], x[8 + b], x[12 + b]);     // over a -> ka, stored at x[4 ka + b]
    x[5] = cmul(x[5], w1);  x[9] = cmul(x[9], w2);   x[13] = cmul(x[13], w3);      // b = 1: ka = 1,2,3
    x[6] = cmul(x[6], w2);  x[10] = cmul(x[10], w4); x[14] = cmul(x[14], w6);      // b = 2
    x[7] = cmul(x[7], w3);  x[11] = cmul(x[11], w6); x[15] = cmul(x[15], w9);      // b = 3
#pragma unroll
    for (int ka = 0; ka < 4; ++ka) fft4(x[4 * ka], x[4 * ka + 1], x[4 * ka + 2], x[4 * ka + 3]);   // over b -> kb
    // element (ka, kb) now sits at x[4 ka + kb]; output index k = ka + 4 kb -> transpose
    Cx<float> t;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = i + 1; j < 4; ++j) { t = x[4 * i + j]; x[4 * i + j] = x[4 * j + i]; x[4 * j + i] = t; }
}

// Frame pool: the reference runs one forward per 10-s window at a 1-s hop (model_loader.py:396-407),
// so a frame whose 1024 samples lie inside a window (frame index 2..998) is recomputed identically
// by up to ten windows.  Here every DISTINCT frame is computed once: pool entry p describes
// (window start sample, valid samples of that window, frame index inside the window); windows then
// address the pool through an index table.  Edge frames (0, 1, 999, 1000: reflect padding / zero
// tail) stay per window.  out: [n_pool, 64] BatchNorm-ed log-mel rows.
__global__ void __launch_bounds__(kClWarps * 32)
clap_logmel_kernel(const int16_t* __restrict__ pcm, const long long* __restrict__ pool_start,
                   const int* __restrict__ pool_valid, const int* __restrict__ pool_frame, long long n_pool,
                   ClapFrontTables tab, float* __restrict__ out /*[n_pool,64]*/)
{
    extern __shared__ __align__(16) unsigned char cl_smem[];
    float* sm = reinterpret_cast<float*>(cl_smem);
    Cx<float>* tw = reinterpret_cast<Cx<float>*>(sm);            // 512 complex
    float* hann = sm + 1024;
    float* melw = hann + kClFft;
    float* bns = melw + kClMel * kClMelTaps;
    float* bnb = bns + kClMel;
    float* wbuf = bnb + kClMel;                                   // per warp: 512 complex + 516 floats
    int* mstart = reinterpret_cast<int*>(wbuf + kClWarps * (1024 + 516));
    int* mcount = mstart + kClMel;
    for (int i = threadIdx.x; i < 512; i += blockDim.x) { tw[i].re = tab.twiddle[2 * i]; tw[i].im = tab.twiddle[2 * i + 1]; }
    for (int i = threadIdx.x; i < kClFft; i += blockDim.x) hann[i] = tab.hann[i];
    for (int i = threadIdx.x; i < kClMel * kClMelTaps; i += blockDim.x) melw[i] = tab.mel_w[i];
    for (int i = threadIdx.x; i < kClMel; i += blockDim.x) {
        mstart[i] = tab.mel_start[i]; mcount[i] = tab.mel_count[i]; bns[i] = tab.bn_scale[i]; bnb[i] = tab.bn_shift[i];
    }
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    Cx<float>* z = reinterpret_cast<Cx<float>*>(wbuf + warp * (1024 + 516));
    float* pw = wbuf + warp * (1024 + 516) + 1024;

    float hw[16][2];
#pragma unroll
    for (int n1 = 0; n1 < 16; ++n1) { const int n = 32 * n1 + lane; hw[n1][0] = hann[2 * n]; hw[n1][1] = hann[2 * n + 1]; }
    Cx<float> tw1[16];
#pragma unroll
    for (int k1 = 0; k1 < 16; ++k1) {
        const int m = 2 * lane * k1;                              // W_512^(lane k1) = W_1024^(2 lane k1)
        const Cx<float> w = tw[m & 511];
        tw1[k1] = (m & 512) ? Cx<float>{-w.re, -w.im} : w;
    }
    Cx<float> tw2[5];
#pragma unroll
    for (int s = 0; s < 5; ++s) { const int h = 16 >> s; tw2[s] = tw[(lane & (h - 1)) * (512 / h)]; }
    const int rev = __brev((unsigned)lane) >> 27;

    const long long total = n_pool;
    for (long long g = (long long)blockIdx.x * kClWarps + warp; g < total; g += (long long)gridDim.x * kClWarps) {
        const int f = pool_frame[g];
        const int16_t* src = pcm + pool_start[g];
        const int valid = pool_valid[g];
        Cx<float> a[16];
#pragma unroll
        for (int n1 = 0; n1 < 16; ++n1) {
            const int n = 32 * n1 + lane;
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                int i = f * kClHop - kClFft / 2 + 2 * n + e;      // centre=True: frame starts 512 before f*hop
                if (i < 0) i = -i;                                // reflect padding of the zero-padded window
                if (i >= kClChunk) i = 2 * (kClChunk - 1) - i;
                v[e] = i < valid ? tab.pcm_lut[(int)src[i] + 32768] : 0.0f;
            }
            a[n1].re = v[0] * hw[n1][0];
            a[n1].im = v[1] * hw[n1][1];
        }
        fft16(a);
#pragma unroll
        for (int k1 = 1; k1 < 16; ++k1) a[k1] = cmul(a[k1], tw1[k1]);
#pragma unroll
        for (int s = 0; s < 5; ++s) {
            const int h = 16 >> s;
            const bool upper = (lane & h) != 0;
#pragma unroll
            for (int r = 0; r < 16; ++r) {
                Cx<float> p = {shfl_xor_t(a[r].re, h), shfl_xor_t(a[r].im, h)};
                a[r] = upper ? cmul(csub(p, a[r]), tw2[s]) : cadd(a[r], p);
            }
        }
#pragma unroll
        for (int k1 = 0; k1 < 16; ++k1) z[k1 + 16 * rev] = a[k1];
        __syncwarp();
        for (int k = lane; k <= 256; k += 32) {
            const Cx<float> x = z[k], y = z[(512 - k) & 511];
            const float er = 0.5f * (x.re + y.re), ei = 0.5f * (x.im - y.im);
            const float orr = 0.5f * (x.im + y.im), oi = -0.5f * (x.re - y.re);
            const Cx<float> w = tw[k & 511];
            const float pr = orr * w.re - oi * w.im, pi = orr * w.im + oi * w.re;
            const float xr = er + pr, xi = ei + pi, yr = er - pr, yi = ei - pi;
            pw[k] = xr * xr + xi * xi;                             // power spectrum
            pw[512 - k] = yr * yr + yi * yi;
        }
        __syncwarp();
        float* dst = out + g * kClMel;
#pragma unroll
        for (int hsel = 0; hsel < 2; ++hsel) {
            const int b = hsel ? 63 - lane : lane;
            const int st = mstart[b], cnt = mcount[b];
            float acc = 0.f;
            for (int i = 0; i < cnt; ++i) acc = fmaf(pw[st + i], melw[b * kClMelTaps + i], acc);
            const float lm = 10.0f * log10f(fmaxf(acc, 1e-10f));
            dst[b] = lm * bns[b] + bnb[b];
        }
        __syncwarp();
    }
}

// cubic convolution coefficients (A = -0.75, as torch's upsample_bicubic2d)
__device__ __forceinline__ void cubic_coeffs(float t, float (&c)[4]) {
    const float A = -0.75f;
    float x = t + 1.0f; c[0] = ((A * x - 5.0f * A) * x + 8.0f * A) * x - 4.0f * A;
    x = t;              c[1] = ((A + 2.0f) * x - (A + 3.0f)) * x * x + 1.0f;
    x = 1.0f - t;       c[2] = ((A + 2.0f) * x - (A + 3.0f)) * x * x + 1.0f;
    x = 2.0f - t;       c[3] = ((A * x - 5.0f * A) * x + 8.0f * A) * x - 4.0f * A;
}

// one warp per token (patch).  lm: frame pool [n_pool,64] (already BatchNorm-ed), addressed through
// frame_index [B][1001]; w: [96][16]; x out: [B,4096,96]
template <int CPL>                                              // channels per lane: embed dim = 32 CPL (96 tiny, 128 base)
__global__ void __launch_bounds__(256)
clap_patch_embed_kernel(const float* __restrict__ lm, const int* __restrict__ frame_index,
                        const float* __restrict__ w, const float* __restrict__ bias,
                        const float* __restrict__ gamma, const float* __restrict__ beta, int n_chunks,
                        float* __restrict__ x)
{
    const int lane = threadIdx.x & 31;
    // the 96x16 filter bank, bias and LayerNorm affine live in registers (3 channels per lane) and are
    // reused for every token this warp handles
    float wr[CPL][16], br[CPL], gr[CPL], ber[CPL];
#pragma unroll
    for (int u = 0; u < CPL; ++u) {
        const int ch = lane + 32 * u;
        br[u] = bias[ch]; gr[u] = gamma[ch]; ber[u] = beta[ch];
        const float4* wp = reinterpret_cast<const float4*>(w + ch * 16);
#pragma unroll
        for (int q4 = 0; q4 < 4; ++q4) {
            const float4 t4 = wp[q4];
            wr[u][4 * q4] = t4.x; wr[u][4 * q4 + 1] = t4.y; wr[u][4 * q4 + 2] = t4.z; wr[u][4 * q4 + 3] = t4.w;
        }
    }
    const long long total = (long long)n_chunks * 4096;
    for (long long tok = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); tok < total; tok += (long long)gridDim.x * 8) {
        const int b = (int)(tok >> 12), p = (int)(tok & 4095);
        const int ph = p >> 6, pwid = p & 63;                          // image row block / col block
        const int j = ph >> 4, f0 = (ph & 15) * 4;                     // time block, first mel bin
        // lanes 0..15: pixel (r = lane / 4 -> mel f0 + r, c = lane % 4 -> time)
        float pix = 0.f;
        if (lane < 16) {
            const int r = lane >> 2, c = lane & 3;
            const int t = j * 256 + pwid * 4 + c;                      // 0..1023 on the resized time axis
            const float s = (float)t * (float)(kClFrames - 1) / 1023.0f;     // align_corners=True
            const int i0 = (int)floorf(s);
            float cf[4];
            cubic_coeffs(s - (float)i0, cf);
            const int* fidx = frame_index + (size_t)b * kClFrames;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                int ti = i0 - 1 + k;
                ti = ti < 0 ? 0 : (ti > kClFrames - 1 ? kClFrames - 1 : ti);
                pix = fmaf(cf[k], lm[(size_t)fidx[ti] * kClMel + f0 + r], pix);
            }
        }
        float o[CPL];
#pragma unroll
        for (int u = 0; u < CPL; ++u) o[u] = br[u];
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            const float v = __shfl_sync(0xffffffffu, pix, q);
#pragma unroll
            for (int u = 0; u < CPL; ++u) o[u] = fmaf(wr[u][q], v, o[u]);
        }
        float s1 = 0.f;
#pragma unroll
        for (int u = 0; u < CPL; ++u) s1 += o[u];
        for (int m = 16; m > 0; m >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, m);
        const float mean = s1 / (32.0f * CPL);
        float s2 = 0.f;
#pragma unroll
        for (int u = 0; u < CPL; ++u) { const float dlt = o[u] - mean; s2 += dlt * dlt; }
        for (int m = 16; m > 0; m >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, m);
        const float rstd = rsqrtf(s2 / (32.0f * CPL) + 1e-5f);
#pragma unroll
        for (int u = 0; u < CPL; ++u) x[tok * (32 * CPL) + lane + 32 * u] = (o[u] - mean) * rstd * gr[u] + ber[u];
    }
}

// mode 0: rows in (shifted-)window order; mode 1: patch-merge gather (output row = (b, i, j) on the
// res/2 grid, features = [x(2i,2j), x(2i+1,2j), x(2i,2j+1), x(2i+1,2j+1)], LayerNorm over 4C).
// L lanes per row, 32 / L rows per warp; every lane keeps CHUNKS float4 pieces of its row in registers
// (piece j of lane l = elements 4 (l + L j) ...), so loads are 16-B and stores 8-B per lane, fully
// coalesced, and a warp has 32/L rows in flight (width = 4 L CHUNKS: 96 -> <3,8>, 192 -> <3,16>, ...).
// out: fp16 [rows, ld_out] (columns >= width zero filled).
template <int CHUNKS, int L>
__global__ void __launch_bounds__(256)
clap_ln_kernel(const float* x, const float* __restrict__ gamma, const float* __restrict__ beta,
               long long n_rows, int C, int ld_out, int res, int shift, int mode, __half* __restrict__ out,
               float* out32 = nullptr /* optional fp32 copy of the normalised row (row order o, stride width); may alias x */,
               int gelu = 0 /* exact-erf GELU after the affine (wav2vec2 "layer" feature encoder) */)
{
    constexpr int R = 32 / L;                                      // rows per warp
    constexpr int width = 4 * L * CHUNKS;
    const int lane = threadIdx.x & 31;
    const int li = lane % L;
    const long long o = ((long long)blockIdx.x * 8 + (threadIdx.x >> 5)) * R + lane / L;
    const bool live = o < n_rows;
    float4 v[CHUNKS];
    if (live) {
        if (mode == 0) {
            const float4* src = reinterpret_cast<const float4*>(x + (res ? window_row_to_token(o, res, shift) : o) * C);   // res = 0: rows as they are
#pragma unroll
            for (int j = 0; j < CHUNKS; ++j) v[j] = src[li + L * j];
        } else {
            const int half = res >> 1;
            const int jx = (int)(o % half);
            const int iy = (int)((o / half) % half);
            const long long b = o / ((long long)half * half);
            const float* base = x + ((b * res + 2 * iy) * res + 2 * jx) * C;
            // concat order x0 | x1 | x2 | x3 = (2i,2j) (2i+1,2j) (2i,2j+1) (2i+1,2j+1); C is a multiple of 4
#pragma unroll
            for (int j = 0; j < CHUNKS; ++j) {
                const int i = 4 * (li + L * j);
                const int part = i / C, c = i - part * C;
                v[j] = *reinterpret_cast<const float4*>(base + (size_t)((part & 1) ? res * C : 0) + ((part & 2) ? C : 0) + c);
            }
        }
    } else {
#pragma unroll
        for (int j = 0; j < CHUNKS; ++j) v[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float s1 = 0.f;
#pragma unroll
    for (int j = 0; j < CHUNKS; ++j) s1 += (v[j].x + v[j].y) + (v[j].z + v[j].w);
#pragma unroll
    for (int m = L / 2; m > 0; m >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, m);
    const float mean = s1 / (float)width;
    float s2 = 0.f;
#pragma unroll
    for (int j = 0; j < CHUNKS; ++j) {
        const float a = v[j].x - mean, b2 = v[j].y - mean, c2 = v[j].z - mean, d2 = v[j].w - mean;
        s2 += (a * a + b2 * b2) + (c2 * c2 + d2 * d2);
    }
#pragma unroll
    for (int m = L / 2; m > 0; m >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, m);
    const float rstd = rsqrtf(s2 / (float)width + 1e-5f);
    if (!live) return;
    __half* dst = out + o * ld_out;
#pragma unroll
    for (int j = 0; j < CHUNKS; ++j) {
        const int i = 4 * (li + L * j);
        const float4 g4 = *reinterpret_cast<const float4*>(gamma + i);
        const float4 b4 = *reinterpret_cast<const float4*>(beta + i);
        float y0 = (v[j].x - mean) * rstd * g4.x + b4.x, y1 = (v[j].y - mean) * rstd * g4.y + b4.y;
        float y2 = (v[j].z - mean) * rstd * g4.z + b4.z, y3 = (v[j].w - mean) * rstd * g4.w + b4.w;
        if (gelu) {
            y0 = 0.5f * y0 * (1.0f + erff(y0 * 0.70710678118654752f)); y1 = 0.5f * y1 * (1.0f + erff(y1 * 0.70710678118654752f));
            y2 = 0.5f * y2 * (1.0f + erff(y2 * 0.70710678118654752f)); y3 = 0.5f * y3 * (1.0f + erff(y3 * 0.70710678118654752f));
        }
        const __half2 h0 = __floats2half2_rn(y0, y1);
        const __half2 h1 = __floats2half2_rn(y2, y3);
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&h0);
        pk.y = *reinterpret_cast<const uint32_t*>(&h1);
        *reinterpret_cast<uint2*>(dst + i) = pk;
        if (out32 != nullptr)                                      // post-LN transformers: the normalised row IS the new stream
            *reinterpret_cast<float4*>(out32 + o * width + i) = make_float4(y0, y1, y2, y3);
    }
    for (int i = width + li; i < ld_out; i += L) dst[i] = __float2half_rn(0.f);
}

// x[token(o)][0:C] += y[o][0:C]   (windowed = 1: o is a window-ordered row)
__global__ void __launch_bounds__(256)
clap_residual_add_kernel(float* __restrict__ x, const float* __restrict__ y, long long n_rows, int C, int ld_y,
                         int res, int shift, int windowed)
{
    const long long total = n_rows * C;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x) {
        const long long o = e / C;
        const int c = (int)(e % C);
        const long long t = windowed ? window_row_to_token(o, res, shift) : o;
        x[t * C + c] += y[o * ld_y + c];
    }
}

// y[o][0:C] -> x[o][0:C]   (patch merging output becomes the new residual stream)
__global__ void __launch_bounds__(256)
clap_copy_rows_kernel(float* __restrict__ x, const float* __restrict__ y, long long n_rows, int C, int ld_y)
{
    const long long total = n_rows * C;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total;
         e += (long long)gridDim.x * blockDim.x)
        x[e] = y[(e / C) * ld_y + (e % C)];
}

// Window attention on the warp-level tensor-core path (mma.sync m16n8k16 / m16n8k8, fp16 in / fp32
// accumulate): a 64 x 64 x 24 problem per (window, head) is far too small for a wgmma tile,
// but maps exactly onto 16x8 fragments.  One warp per (window, head):
//   staging  Q, K, V rows (24 halves = 48 B each) with 16-B cp.async into warp-private smem, row
//            stride 48 B: conflict-free for the fragment loads below and for ldmatrix
//   S = Q K^T            4 m-tiles x 8 n-tiles, head dim 24 = one k16 + one k8 step
//   S = S/sqrt(24) + relative-position bias (+ -100 across shift regions); row softmax in registers
//   O = P V              per m-tile 3 n-tiles x 4 k-steps, P re-used straight from the S accumulators,
//                        V fragments by ldmatrix.trans from the row-major tile
// qkv: fp16 [rows, ld] with q | k | v at column offsets 0, C, 2C and head h at h*24.
// relbias: fp32 [heads][64][64].  out: fp16 [rows, ld_out] (head h at h*24).
constexpr int kAttWarps = 4;
constexpr int kAttStages = 1;     // 2 = prefetch the next unit into a second warp-private buffer: measured SLOWER
                                  // (12 instead of 20 resident warps per SM: 122 vs 110 ms per 3 steps), kept for reference
// head dim 24 (HTSAT-tiny): rows of 48 B; head dim 32 (HTSAT-base): rows padded to 80 B - both strides keep the
// 32-bit fragment loads and ldmatrix conflict-free and 16-B aligned for cp.async
__host__ __device__ constexpr int att_row_halves(int hd) { return hd == 24 ? 24 : 40; }
__host__ __device__ constexpr int att_smem_bytes(int hd, int warps, int stages) { return warps * stages * 3 * 64 * att_row_halves(hd) * 2; }

__device__ __forceinline__ void mma_m16n8k8(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t b0) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(b0));
}
__device__ __forceinline__ uint32_t pack_h2(float x, float y) {
    __half2 h = __floats2half2_rn(x, y);
    return *reinterpret_cast<uint32_t*>(&h);
}

template <int HD>
__global__ void __launch_bounds__(kAttWarps * 32)
clap_window_attention_kernel(const __half* __restrict__ qkv, int ld, int C, int heads,
                             const float* __restrict__ relbias, int res, int shift, long long n_windows,
                             __half* __restrict__ out, int ld_out)
{
    constexpr int kAttRow = att_row_halves(HD);
    constexpr int kAttMat = 64 * kAttRow;
    constexpr int kVec = HD / 8;                                   // 16-B vectors per row
    constexpr int kNT = HD / 8;                                    // PV n-tiles
    extern __shared__ __align__(16) unsigned char att_smem[];           // [warps][stages][Q | K | V], row-major [64][24] each
    __half* tiles_base = reinterpret_cast<__half*>(att_smem);
    __shared__ int rid[kAttWarps][64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane >> 2, t = lane & 3;
    const long long units = n_windows * heads;
    const int lg_nw = 28 - __clz(res);
    const int nw = res >> 3;
    const float scale = HD == 24 ? 0.20412414523193151f : 0.17677669529663689f;   // 1 / sqrt(head dim)
    __half* my_tiles = tiles_base + (size_t)warp * kAttStages * 3 * kAttMat;
    const uint32_t tiles_u32 = (uint32_t)__cvta_generic_to_shared(my_tiles);
    // 3 matrices x 64 rows x kVec vectors of 16 B = 6 kVec cp.async per lane
    auto fetch = [&](long long unit, int stage) {
        const long long w_ = unit / heads;
        const int h_ = (int)(unit - w_ * heads);
        const __half* base = qkv + w_ * 64 * ld + h_ * HD;
        const uint32_t t32 = tiles_u32 + stage * 3 * kAttMat * 2;
#pragma unroll
        for (int it = 0; it < 6 * kVec; ++it) {
            const int i = it * 32 + lane;
            const int mtx = i / (64 * kVec), rem = i - mtx * (64 * kVec);
            const int r = rem / kVec, v = rem - r * kVec;
            const uint32_t dst = t32 + ((mtx * 64 + r) * kAttRow + v * 8) * 2;
            const __half* src = base + (size_t)r * ld + mtx * C + v * 8;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst), "l"(src));
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    const long long stride = (long long)gridDim.x * kAttWarps;
    long long u = (long long)blockIdx.x * kAttWarps + warp;
    if (kAttStages == 2 && u < units) fetch(u, 0);
    for (int stage = 0; u < units; u += stride, stage ^= (kAttStages - 1)) {
        const long long win = u / heads;
        const int h = (int)(u - win * heads);
        const __half* q_s = my_tiles + stage * 3 * kAttMat;
        const __half* k_s = q_s + kAttMat;
        const uint32_t tile_u32 = tiles_u32 + stage * 3 * kAttMat * 2;
        // ldmatrix.trans row addresses for the V fragments: lanes 0-7 / 8-15 give the key rows of the
        // two 8x8 blocks of one n-tile (b0, b1), lanes 16-31 the same rows of the next n-tile
        const uint32_t v_ld = tile_u32 + 2 * kAttMat * 2 + ((lane & 15) * kAttRow + (lane >> 4) * 8) * 2;
        if (kAttStages == 2) {                      // next unit -> other buffer (free: its reader finished an iteration ago)
            if (u + stride < units) fetch(u + stride, stage ^ 1);
            else asm volatile("cp.async.commit_group;" ::: "memory");
        } else {
            fetch(u, 0);
        }
        if (shift) {
            const int wx = (int)win & (nw - 1), wy = (int)(win >> lg_nw) & (nw - 1);
            for (int i = lane; i < 64; i += 32) {
                const int y = wy * 8 + (i >> 3), xx = wx * 8 + (i & 7);   // coordinates in the SHIFTED image
                const int ry = y < res - 8 ? 0 : (y < res - shift ? 1 : 2);
                const int rx = xx < res - 8 ? 0 : (xx < res - shift ? 1 : 2);
                rid[warp][i] = ry * 3 + rx;
            }
        }
        if (kAttStages == 2) asm volatile("cp.async.wait_group 1;" ::: "memory");
        else asm volatile("cp.async.wait_all;" ::: "memory");
        __syncwarp();
        const float* bias_h = relbias + (size_t)h * 64 * 64;
#pragma unroll 1
        for (int mt = 0; mt < 4; ++mt) {
            const int r0 = mt * 16 + g, r1 = r0 + 8;
            // relative-position bias of this m-tile: issue the 16 loads before the MMAs so their latency
            // is hidden (ncu: the scale+bias FFMAs were the top long-scoreboard stall)
            float2 bias0[8], bias1[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                bias0[j] = __ldg(reinterpret_cast<const float2*>(bias_h + r0 * 64 + j * 8 + 2 * t));
                bias1[j] = __ldg(reinterpret_cast<const float2*>(bias_h + r1 * 64 + j * 8 + 2 * t));
            }
            float sacc[8][4];
#pragma unroll
            for (int j = 0; j < 8; ++j) { sacc[j][0] = sacc[j][1] = sacc[j][2] = sacc[j][3] = 0.f; }
            {
                const uint32_t a0 = *reinterpret_cast<const uint32_t*>(q_s + r0 * kAttRow + 2 * t);
                const uint32_t a1 = *reinterpret_cast<const uint32_t*>(q_s + r1 * kAttRow + 2 * t);
                const uint32_t a2 = *reinterpret_cast<const uint32_t*>(q_s + r0 * kAttRow + 2 * t + 8);
                const uint32_t a3 = *reinterpret_cast<const uint32_t*>(q_s + r1 * kAttRow + 2 * t + 8);
                const uint32_t a4 = *reinterpret_cast<const uint32_t*>(q_s + r0 * kAttRow + 2 * t + 16);
                const uint32_t a5 = *reinterpret_cast<const uint32_t*>(q_s + r1 * kAttRow + 2 * t + 16);
                uint32_t a6 = 0, a7 = 0;
                if (HD == 32) {
                    a6 = *reinterpret_cast<const uint32_t*>(q_s + r0 * kAttRow + 2 * t + 24);
                    a7 = *reinterpret_cast<const uint32_t*>(q_s + r1 * kAttRow + 2 * t + 24);
                }
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const __half* kr = k_s + (j * 8 + g) * kAttRow + 2 * t;
                    const uint32_t b0 = *reinterpret_cast<const uint32_t*>(kr);
                    const uint32_t b1 = *reinterpret_cast<const uint32_t*>(kr + 8);
                    const uint32_t b2 = *reinterpret_cast<const uint32_t*>(kr + 16);
                    mma_m16n8k16(sacc[j], a0, a1, a2, a3, b0, b1);
                    if (HD == 24) mma_m16n8k8(sacc[j], a4, a5, b2);
                    else mma_m16n8k16(sacc[j], a4, a5, a6, a7, b2, *reinterpret_cast<const uint32_t*>(kr + 24));
                }
            }
            // scale + bias + mask, row max
            const int id0 = shift ? rid[warp][r0] : 0, id1 = shift ? rid[warp][r1] : 0;
            float mx0 = -3.0e38f, mx1 = -3.0e38f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = j * 8 + 2 * t;
                const float2 b0v = bias0[j], b1v = bias1[j];
                sacc[j][0] = sacc[j][0] * scale + b0v.x; sacc[j][1] = sacc[j][1] * scale + b0v.y;
                sacc[j][2] = sacc[j][2] * scale + b1v.x; sacc[j][3] = sacc[j][3] * scale + b1v.y;
                if (shift) {
                    const int ic0 = rid[warp][c], ic1 = rid[warp][c + 1];
                    if (ic0 != id0) sacc[j][0] -= 100.0f;
                    if (ic1 != id0) sacc[j][1] -= 100.0f;
                    if (ic0 != id1) sacc[j][2] -= 100.0f;
                    if (ic1 != id1) sacc[j][3] -= 100.0f;
                }
                mx0 = fmaxf(mx0, fmaxf(sacc[j][0], sacc[j][1]));
                mx1 = fmaxf(mx1, fmaxf(sacc[j][2], sacc[j][3]));
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                sacc[j][0] = __expf(sacc[j][0] - mx0); sacc[j][1] = __expf(sacc[j][1] - mx0);
                sacc[j][2] = __expf(sacc[j][2] - mx1); sacc[j][3] = __expf(sacc[j][3] - mx1);
                sum0 += sacc[j][0] + sacc[j][1];
                sum1 += sacc[j][2] + sacc[j][3];
            }
            sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
            sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
            const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
            // O = P V : P fragments come straight from the (normalised) S accumulators
            float oacc[kNT][4];
#pragma unroll
            for (int n = 0; n < kNT; ++n) { oacc[n][0] = oacc[n][1] = oacc[n][2] = oacc[n][3] = 0.f; }
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t a0 = pack_h2(sacc[2 * kk][0] * inv0, sacc[2 * kk][1] * inv0);
                const uint32_t a1 = pack_h2(sacc[2 * kk][2] * inv1, sacc[2 * kk][3] * inv1);
                const uint32_t a2 = pack_h2(sacc[2 * kk + 1][0] * inv0, sacc[2 * kk + 1][1] * inv0);
                const uint32_t a3 = pack_h2(sacc[2 * kk + 1][2] * inv1, sacc[2 * kk + 1][3] * inv1);
                uint32_t b[8];
                const uint32_t va = v_ld + kk * 16 * kAttRow * 2;
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(b[0]), "=r"(b[1]), "=r"(b[2]), "=r"(b[3]) : "r"(va));
                if (HD == 24) {
                    asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];"
                                 : "=r"(b[4]), "=r"(b[5]) : "r"(va + ((lane >> 4) ? -16 : 32)));   // dims 16..23 (lanes >= 16: address unused but valid)
                } else {
                    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                                 : "=r"(b[4]), "=r"(b[5]), "=r"(b[6]), "=r"(b[7]) : "r"(va + 32));   // dims 16..31
                }
#pragma unroll
                for (int n = 0; n < kNT; ++n) mma_m16n8k16(oacc[n], a0, a1, a2, a3, b[2 * n], b[2 * n + 1]);
            }
            __half* d0 = out + (win * 64 + r0) * ld_out + h * HD;
            __half* d1 = out + (win * 64 + r1) * ld_out + h * HD;
#pragma unroll
            for (int n = 0; n < kNT; ++n) {
                *reinterpret_cast<uint32_t*>(d0 + n * 8 + 2 * t) = pack_h2(oacc[n][0], oacc[n][1]);
                *reinterpret_cast<uint32_t*>(d1 + n * 8 + 2 * t) = pack_h2(oacc[n][2], oacc[n][3]);
            }
        }
        __syncwarp();
    }
}

// one block (256 threads) per chunk: LayerNorm(768) of the 64 tokens, mean over tokens,
// 768 -> 512 ReLU -> 512, L2 normalise, fp16 out [B, 512]
template <int D>                                                // final width: 768 (tiny) or 1024 (base)
__global__ void __launch_bounds__(256)
clap_head_kernel(const float* __restrict__ x /*[B,64,D]*/, const float* __restrict__ gamma,
                 const float* __restrict__ beta, const float* __restrict__ w1, const float* __restrict__ b1,
                 const float* __restrict__ w2, const float* __restrict__ b2, __half* __restrict__ out)
{
    __shared__ float pooled[D];
    __shared__ float part[8][D];                                 // per-warp partial means (fixed-order reduce)
    __shared__ float h1[512];
    __shared__ float h2[512];
    __shared__ float red[8];
    const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int E = D / 32;
    float acc_tok[E];
#pragma unroll
    for (int k = 0; k < E; ++k) acc_tok[k] = 0.f;
    for (int t = warp; t < 64; t += 8) {
        const float* row = x + ((size_t)b * 64 + t) * D;
        float v[E];
        float s1 = 0.f;
#pragma unroll
        for (int k = 0; k < E; ++k) { v[k] = row[lane + 32 * k]; s1 += v[k]; }
        for (int m = 16; m > 0; m >>= 1) s1 += __shfl_xor_sync(0xffffffffu, s1, m);
        const float mean = s1 / (float)D;
        float s2 = 0.f;
#pragma unroll
        for (int k = 0; k < E; ++k) { const float dlt = v[k] - mean; s2 += dlt * dlt; }
        for (int m = 16; m > 0; m >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, m);
        const float rstd = rsqrtf(s2 / (float)D + 1e-5f);
#pragma unroll
        for (int k = 0; k < E; ++k) {
            const int c = lane + 32 * k;
            acc_tok[k] += (v[k] - mean) * rstd * gamma[c] + beta[c];
        }
    }
#pragma unroll
    for (int k = 0; k < E; ++k) part[warp][lane + 32 * k] = acc_tok[k];
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += 256) {
        float sacc = 0.f;
#pragma unroll
        for (int wv = 0; wv < 8; ++wv) sacc += part[wv][i];
        pooled[i] = sacc * (1.0f / 64.0f);
    }
    __syncthreads();
    for (int o = warp; o < 512; o += 8) {
        float acc = 0.f;
        for (int k = lane; k < D; k += 32) acc = fmaf(w1[(size_t)o * D + k], pooled[k], acc);
        for (int m = 16; m > 0; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
        if (lane == 0) h1[o] = fmaxf(acc + b1[o], 0.f);
    }
    __syncthreads();
    float sq = 0.f;
    for (int o = warp; o < 512; o += 8) {
        float acc = 0.f;
        for (int k = lane; k < 512; k += 32) acc = fmaf(w2[(size_t)o * 512 + k], h1[k], acc);
        for (int m = 16; m > 0; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
        if (lane == 0) { h2[o] = acc + b2[o]; sq += h2[o] * h2[o]; }
    }
    if (lane == 0) red[warp] = sq;
    __syncthreads();
    float tot = 0.f;
    for (int k = 0; k < 8; ++k) tot += red[k];
    const float inv = 1.0f / fmaxf(sqrtf(tot), 1e-12f);            // F.normalize eps
    for (int i = threadIdx.x; i < 512; i += 256) out[(size_t)b * 512 + i] = __float2half_rn(h2[i] * inv);
}

}  // namespace fad
