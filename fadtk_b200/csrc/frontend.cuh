// VGGish front-end on the GPU: PCM16 -> log-mel examples, and the first convolution.
//
//  logmel_kernel   int16 PCM -> /32768 -> 25 ms periodic-Hann frames (hop 10 ms) -> |rFFT_512|
//                  -> 64 HTK-mel bands (125..7500 Hz) -> log(x + 0.01) -> fp32 [B, 96, 64].
//                  Replaces torchvggish's numpy front-end reached from
//                  fadtk/model_loader.py:107-108 (+ load_wav :63-70); SURVEY.md appendix A K1/K2.
//                  One warp per STFT frame: the 512-point real FFT is a 256-point complex FFT
//                  factored 8 x 32 - an 8-point FFT in registers, twiddles, then a 32-point FFT
//                  across the lanes with shuffles - so shared memory is touched once, for the
//                  real-FFT split and the sparse mel filters.  <3 % of the model FLOPs, feeds a
//                  log(): full precision on the CUDA cores.  T = float (default) moves the FAD by
//                  <= 1.5e-6 relative vs the reference's float64 numpy (CPU experiment, DESIGN.md);
//                  T = double matches float64 to 2e-6 in the fp32 output.
//  conv1_kernel    3x3 conv 1->64 + bias + ReLU + 2x2 max-pool on fp32 input (K = 9 is too thin
//                  for the tensor pipe); writes NHWC fp16 [B, 48, 32, 64] for the wgmma layers.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace fad {

constexpr int kWin = 400, kHop = 160, kFft = 512, kBins = 257, kMel = 64, kExFrames = 96;
constexpr int kMelMaxTaps = 24;          // widest triangular filter spans < 24 FFT bins
constexpr int kFeWarps = 8;

// Host-built tables (double precision, converted on upload).
struct FrontendTables {
    const double* twiddle;   // [256][2]  exp(-2 pi i k / 512)
    const double* hann;      // [400]
    const double* mel_w;     // [64][kMelMaxTaps]
    const int* mel_start;    // [64] first FFT bin with non-zero weight
    const int* mel_count;    // [64]
};

template <typename T> struct Cx { T re, im; };

template <typename T>
__host__ __device__ constexpr size_t logmel_smem_bytes() {
    return sizeof(T) * (size_t)(kFeWarps * (2 * 256 + 260) + 2 * 256 + kWin + kMel * kMelMaxTaps)
         + sizeof(int) * 2 * kMel;
}

// ---- warp-level 256-point complex FFT: 256 = 8 (registers) x 32 (lanes, shuffles) ----------
template <typename T> __device__ __forceinline__ Cx<T> cmul(Cx<T> a, Cx<T> b) {
    return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re};
}
template <typename T> __device__ __forceinline__ Cx<T> cadd(Cx<T> a, Cx<T> b) { return {a.re + b.re, a.im + b.im}; }
template <typename T> __device__ __forceinline__ Cx<T> csub(Cx<T> a, Cx<T> b) { return {a.re - b.re, a.im - b.im}; }
template <typename T> __device__ __forceinline__ Cx<T> mul_neg_i(Cx<T> a) { return {a.im, -a.re}; }   // a * (-i)

// natural-order in, natural-order out, forward transform (e^{-2 pi i nk/8})
template <typename T> __device__ __forceinline__ void fft8(Cx<T> (&a)[8]) {
    const T c = (T)0.70710678118654752440;
    Cx<T> b0 = cadd(a[0], a[4]), b4 = csub(a[0], a[4]);
    Cx<T> b1 = cadd(a[1], a[5]), t1 = csub(a[1], a[5]);
    Cx<T> b2 = cadd(a[2], a[6]), b6 = mul_neg_i(csub(a[2], a[6]));
    Cx<T> b3 = cadd(a[3], a[7]), t3 = csub(a[3], a[7]);
    Cx<T> b5 = {c * (t1.re + t1.im), c * (t1.im - t1.re)};          // * W8^1 = c(1 - i)
    Cx<T> b7 = {c * (t3.im - t3.re), -c * (t3.re + t3.im)};         // * W8^3 = -c(1 + i)
    // even outputs: FFT4(b0,b1,b2,b3); odd outputs: FFT4(b4,b5,b6,b7)
    Cx<T> q0 = cadd(b0, b2), q1 = cadd(b1, b3), q2 = csub(b0, b2), q3 = mul_neg_i(csub(b1, b3));
    a[0] = cadd(q0, q1); a[4] = csub(q0, q1); a[2] = cadd(q2, q3); a[6] = csub(q2, q3);
    Cx<T> r0 = cadd(b4, b6), r1 = cadd(b5, b7), r2 = csub(b4, b6), r3 = mul_neg_i(csub(b5, b7));
    a[1] = cadd(r0, r1); a[5] = csub(r0, r1); a[3] = cadd(r2, r3); a[7] = csub(r2, r3);
}

__device__ __forceinline__ float shfl_xor_t(float v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }
__device__ __forceinline__ double shfl_xor_t(double v, int m) { return __shfl_xor_sync(0xffffffffu, v, m); }

template <typename T>
__global__ void __launch_bounds__(kFeWarps * 32)
logmel_kernel(const int16_t* __restrict__ pcm, const long long* __restrict__ ex_start,
              int n_examples, FrontendTables tab, float* __restrict__ out)
{
    extern __shared__ __align__(16) unsigned char fe_smem[];
    T* sm = reinterpret_cast<T*>(fe_smem);
    Cx<T>* tw = reinterpret_cast<Cx<T>*>(sm);                 // 256 complex: exp(-2 pi i k / 512)
    T* hann = sm + 512;                                        // 400
    T* melw = hann + kWin;                                     // 64*24
    T* wbuf = melw + kMel * kMelMaxTaps;                       // per-warp: 256 complex + 260 mags
    int* mstart = reinterpret_cast<int*>(wbuf + kFeWarps * (512 + 260));
    int* mcount = mstart + kMel;

    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        tw[i].re = (T)tab.twiddle[2 * i]; tw[i].im = (T)tab.twiddle[2 * i + 1];
    }
    for (int i = threadIdx.x; i < kWin; i += blockDim.x) hann[i] = (T)tab.hann[i];
    for (int i = threadIdx.x; i < kMel * kMelMaxTaps; i += blockDim.x) melw[i] = (T)tab.mel_w[i];
    for (int i = threadIdx.x; i < kMel; i += blockDim.x) { mstart[i] = tab.mel_start[i]; mcount[i] = tab.mel_count[i]; }
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    Cx<T>* z = reinterpret_cast<Cx<T>*>(wbuf + warp * (512 + 260));
    T* mag = wbuf + warp * (512 + 260) + 512;

    // per-lane constants: window taps, W_256^(lane*k1), W_32^(lane mod h) for h = 16..1
    T hw[7][2];
#pragma unroll
    for (int n1 = 0; n1 < 7; ++n1) {
        const int n = 32 * n1 + lane;
        hw[n1][0] = n < kWin / 2 ? hann[2 * n] * (T)(1.0 / 32768.0) : (T)0;
        hw[n1][1] = n < kWin / 2 ? hann[2 * n + 1] * (T)(1.0 / 32768.0) : (T)0;
    }
    Cx<T> tw1[8];
#pragma unroll
    for (int k1 = 0; k1 < 8; ++k1) {
        const int m = 2 * lane * k1;                           // W_256^(lane k1) = W_512^(2 lane k1)
        const Cx<T> w = tw[m & 255];
        tw1[k1] = (m & 256) ? Cx<T>{-w.re, -w.im} : w;
    }
    Cx<T> tw2[5];
#pragma unroll
    for (int s = 0; s < 5; ++s) {
        const int h = 16 >> s;
        tw2[s] = tw[(lane & (h - 1)) * (256 / h)];             // W_{2h}^(lane mod h) = W_512^(256/h * ..)
    }
    const int rev = __brev((unsigned)lane) >> 27;              // 5-bit reversal

    const long long total = (long long)n_examples * kExFrames;
    for (long long g = (long long)blockIdx.x * kFeWarps + warp; g < total;
         g += (long long)gridDim.x * kFeWarps) {
        const int e = (int)(g / kExFrames), f = (int)(g % kExFrames);
        const int16_t* src = pcm + ex_start[e] + (long long)f * kHop;

        // z[n] = w[2n] x[2n] + i w[2n+1] x[2n+1], n = 32 n1 + lane (n >= 200 is zero padding)
        Cx<T> a[8];
#pragma unroll
        for (int n1 = 0; n1 < 7; ++n1) {
            const int n = 32 * n1 + lane;
            if (n < kWin / 2) {
                a[n1].re = (T)src[2 * n] * hw[n1][0];
                a[n1].im = (T)src[2 * n + 1] * hw[n1][1];
            } else { a[n1].re = 0; a[n1].im = 0; }
        }
        a[7].re = 0; a[7].im = 0;
        fft8(a);                                               // over n1 -> k1
#pragma unroll
        for (int k1 = 1; k1 < 8; ++k1) a[k1] = cmul(a[k1], tw1[k1]);
        // 32-point DIF across lanes (n2 = lane -> k2, bit-reversed lane order)
#pragma unroll
        for (int s = 0; s < 5; ++s) {
            const int h = 16 >> s;
            const bool upper = (lane & h) != 0;
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                Cx<T> p = {shfl_xor_t(a[r].re, h), shfl_xor_t(a[r].im, h)};
                a[r] = upper ? cmul(csub(p, a[r]), tw2[s]) : cadd(a[r], p);
            }
        }
        // lane holds Z[k1 + 8 k2], k2 = rev(lane)
#pragma unroll
        for (int k1 = 0; k1 < 8; ++k1) z[k1 + 8 * rev] = a[k1];
        __syncwarp();
        // split the packed transform into the 257 bins of the real FFT; keep magnitudes
        for (int k = lane; k <= 128; k += 32) {
            const Cx<T> x = z[k], y = z[(256 - k) & 255];
            const T er = (T)0.5 * (x.re + y.re), ei = (T)0.5 * (x.im - y.im);      // even part
            const T orr = (T)0.5 * (x.im + y.im), oi = (T)-0.5 * (x.re - y.re);    // odd part
            const Cx<T> w = tw[k & 255];
            const T pr = orr * w.re - oi * w.im, pi = orr * w.im + oi * w.re;
            const T xr = er + pr, xi = ei + pi, yr = er - pr, yi = ei - pi;
            mag[k] = sqrt(xr * xr + xi * xi);
            mag[256 - k] = sqrt(yr * yr + yi * yi);
        }
        __syncwarp();
        float* dst = out + g * kMel;
#pragma unroll
        for (int hsel = 0; hsel < 2; ++hsel) {
            const int b = hsel ? 63 - lane : lane;             // pair a narrow and a wide filter per lane
            const int st = mstart[b], cnt = mcount[b];
            T acc = 0;
            for (int i = 0; i < cnt; ++i) acc += mag[st + i] * melw[b * kMelMaxTaps + i];
            dst[b] = (float)log(acc + (T)0.01);
        }
        __syncwarp();
    }
}

// warp-level fp16 x fp16 -> fp32 MMA, C += A[16 x 16] B[16 x 8] (the attention kernels of clap.cuh and whisper.cuh)
__device__ __forceinline__ void mma_m16n8k16(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                             uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// conv1: grid = (6 strips, B); block = 256 threads.  Lane = output-channel pair, warp loops
// over pooled pixels of an 8-row strip; the fp32 input strip (with halo) sits in smem.
__global__ void __launch_bounds__(256)
conv1_kernel(const float* __restrict__ logmel /*[B,96,64]*/, const float* __restrict__ w /*[64,9]*/,
             const float* __restrict__ bias, __half* __restrict__ out /*[B,48,32,64]*/)
{
    __shared__ float tile[18][68];
    const int e = blockIdx.y, strip = blockIdx.x;          // strip: pooled rows [8*strip, 8*strip+8)
    const int row0 = strip * 16 - 1;                       // first input row held (halo)
    const float* src = logmel + (size_t)e * 96 * 64;
    for (int i = threadIdx.x; i < 18 * 66; i += 256) {
        const int r = i / 66, c = i % 66;
        const int gr = row0 + r, gc = c - 1;
        tile[r][c] = (gr >= 0 && gr < 96 && gc >= 0 && gc < 64) ? src[gr * 64 + gc] : 0.0f;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float w0[9], w1[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) { w0[i] = w[(2 * lane) * 9 + i]; w1[i] = w[(2 * lane + 1) * 9 + i]; }
    const float b0 = bias[2 * lane], b1 = bias[2 * lane + 1];
    __syncthreads();

    const int py = warp;                                   // pooled row inside the strip
#pragma unroll 2
    for (int px = 0; px < 32; ++px) {
        float patch[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) patch[r][c] = tile[2 * py + r][2 * px + c];
        float m0 = -3.0e38f, m1 = -3.0e38f;
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                float a0 = 0.f, a1 = 0.f;
#pragma unroll
                for (int kh = 0; kh < 3; ++kh)
#pragma unroll
                    for (int kw = 0; kw < 3; ++kw) {
                        const float x = patch[dy + kh][dx + kw];
                        a0 = fmaf(w0[kh * 3 + kw], x, a0);
                        a1 = fmaf(w1[kh * 3 + kw], x, a1);
                    }
                m0 = fmaxf(m0, a0); m1 = fmaxf(m1, a1);
            }
        m0 = fmaxf(m0 + b0, 0.f); m1 = fmaxf(m1 + b1, 0.f);
        const size_t pix = ((size_t)e * 48 + strip * 8 + py) * 32 + px;
        *reinterpret_cast<__half2*>(out + pix * 64 + 2 * lane) = __floats2half2_rn(m0, m1);
    }
}

}  // namespace fad
