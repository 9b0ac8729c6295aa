// Frechet distance between two Gaussians on the GPU, fp64.
//
//   FAD = |mu1 - mu2|^2 + tr C1 + tr C2 - 2 tr sqrt(C1 C2)
//
// The reference (fadtk/fad.py:88-120) evaluates tr sqrt(C1 C2) through a non-symmetric
// eigen-decomposition V sqrt(D) V^-1 of C1 C2 (LAPACK dgeev + zgetri) - and scipy sqrtm for a
// warning.  Here the eigenvalues of C1 C2 are obtained from the similar SYMMETRIC PSD matrix
//   M = C1^(1/2) C2 C1^(1/2),      tr sqrt(C1 C2) = tr sqrt(M),
// and both square roots come from the coupled Newton-Schulz iteration
//   Y0 = A / |A|_F, Z0 = I;   W = 1.5 I - 0.5 Z Y;   Y <- Y W;   Z <- W Z;   Y -> (A/|A|_F)^(1/2)
// which is nothing but a chain of d x d x d GEMMs.  Zero eigenvalues (rank-deficient covariances,
// n < d) stay exactly zero in Y, so singular inputs need no eps-regularisation branch.
// C1^(1/2) of the baseline can be cached and reused by FAD-inf / per-song scoring.
//
// All scalars (norms, traces) stay on the device; the chain is launched without host syncs.
#pragma once
#include <stdint.h>

namespace fad {

// C = alpha * A * B + beta_diag * I   (row-major d x d, fp64), optional trace(C) accumulation.
// Up to two independent problems per launch (blockIdx.z): the Y <- Y W and Z <- W Z updates of
// one Newton-Schulz iteration run side by side.  64 x 64 tile / 256 threads on DMMA (dgemm_tile below).
//
// Convergence control without host round trips: a launch whose `dev_in` (max |W - I| of the previous
// iteration) is below `tol` returns immediately, so a fixed-length launch sequence costs only
// launch latency once the iteration has converged.  `dev_out` receives max |C - I| (float bits,
// atomicMax), `dev_clear` is zeroed for a later iteration (three rotating slots, see host code).
struct DgemmProblem { const double* A; const double* B; double* C; double alpha, beta_diag; double* trace_out; };
struct DgemmBatch {
    DgemmProblem p[2];
    const float* dev_in; float* dev_out; float* dev_clear; float tol;
};

// One 64 x 64 tile of C = alpha A B + beta_diag I per 256-thread CTA on the FP64 TENSOR pipe
// (mma.sync m8n8k4 f64 -> SASS DMMA.8x8x4, the fp64 MMA shape of sm_90a; wgmma has no f64 kind).
// Returns max |C - I| over this thread's outputs and its share of tr C.
// Layout: 8 warps as 2 (M) x 4 (N); a warp owns 32 x 16 outputs = 4 x 2 DMMA blocks (16 fp64 accumulators
// per thread).  Per 4-wide k-step a warp issues 6 conflict-free LDS.64 (4 A + 2 B fragments) for 8 DMMAs,
// so the tensor pipe and not shared memory is the limit (the CUDA-core tile this replaces needed 6 LDS.128
// per 32 DFMAs and reached 3 TFLOP/s).  Operand tiles keep their global orientation in shared memory -
// A as [m][k] with pitch 20, B as [k][n] with pitch 68 doubles: for the m8n8k4 fragments (A: lane -> row
// lane/4, k lane%4; B: k lane%4, col lane/4) both pitches are = 4 mod 16, i.e. every half-warp touches 16
// distinct 8-byte banks.  Global loads of chunk c+1 are issued before the DMMAs of chunk c (register
// staging, two smem buffers, one barrier per 16-wide K chunk).  Accumulation order is fixed: results are
// bit-reproducible run to run.
constexpr int kDgTileM = 64, kDgTileN = 64, kDgKC = 16;
constexpr int kDgPitchA = kDgKC + 4, kDgPitchB = kDgTileN + 4;

__device__ __forceinline__ void dmma_884(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__device__ __forceinline__ void dgemm_tile(const double* __restrict__ A, const double* __restrict__ B,
                                           double* __restrict__ C, int d, double alpha, double beta_diag,
                                           float& dev, double& tr)
{
    __shared__ __align__(16) double As[2][kDgTileM][kDgPitchA];
    __shared__ __align__(16) double Bs[2][kDgKC][kDgPitchB];
    const int bi = blockIdx.y * kDgTileM, bj = blockIdx.x * kDgTileN;
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;      // warp tile origin inside the CTA tile
    const int fr = lane >> 2, fk = lane & 3;                    // fragment coordinates
    // loader roles: A chunk = 64 rows x 16 k (4 consecutive k per thread), B chunk = 16 k x 64 cols (4 cols per thread)
    const int la_row = t >> 2, la_k = (t & 3) * 4, lb_k = t >> 4, lb_c = (t & 15) * 4;
    // 16-B vector path: 4-groups are then entirely inside or outside the matrix
    const bool vec = (d & 3) == 0 && ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B) |
                                       reinterpret_cast<uintptr_t>(C)) & 15) == 0;
    const bool a_row_ok = bi + la_row < d;
    const double* a_src = A + (size_t)(bi + la_row) * d + la_k;
    double ra[4], rb[4];
    auto fetch = [&](int k0) {
        const double* b_src = B + (size_t)(k0 + lb_k) * d + bj + lb_c;
        const bool kok = k0 + lb_k < d;
        if (vec) {
            double2 v0 = make_double2(0.0, 0.0), v1 = v0, w0 = v0, w1 = v0;
            if (a_row_ok && k0 + la_k < d) {
                v0 = *reinterpret_cast<const double2*>(a_src + k0);
                v1 = *reinterpret_cast<const double2*>(a_src + k0 + 2);
            }
            if (kok && bj + lb_c < d) {
                w0 = *reinterpret_cast<const double2*>(b_src);
                w1 = *reinterpret_cast<const double2*>(b_src + 2);
            }
            ra[0] = v0.x; ra[1] = v0.y; ra[2] = v1.x; ra[3] = v1.y;
            rb[0] = w0.x; rb[1] = w0.y; rb[2] = w1.x; rb[3] = w1.y;
        } else {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                ra[e] = (a_row_ok && k0 + la_k + e < d) ? a_src[k0 + e] : 0.0;
                rb[e] = (kok && bj + lb_c + e < d) ? b_src[e] : 0.0;
            }
        }
    };
    auto stage = [&](int buf) {
        *reinterpret_cast<double2*>(&As[buf][la_row][la_k]) = make_double2(ra[0], ra[1]);
        *reinterpret_cast<double2*>(&As[buf][la_row][la_k + 2]) = make_double2(ra[2], ra[3]);
        *reinterpret_cast<double2*>(&Bs[buf][lb_k][lb_c]) = make_double2(rb[0], rb[1]);
        *reinterpret_cast<double2*>(&Bs[buf][lb_k][lb_c + 2]) = make_double2(rb[2], rb[3]);
    };
    double c[4][2][2] = {};
    const int chunks = (d + kDgKC - 1) / kDgKC;
    fetch(0);
    stage(0);
    __syncthreads();
    for (int ch = 0; ch < chunks; ++ch) {
        const int buf = ch & 1;
        if (ch + 1 < chunks) fetch((ch + 1) * kDgKC);
#pragma unroll
        for (int kk = 0; kk < kDgKC; kk += 4) {
            double a[4], b[2];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[buf][wm + i * 8 + fr][kk + fk];
#pragma unroll
            for (int j = 0; j < 2; ++j) b[j] = Bs[buf][kk + fk][wn + j * 8 + fr];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j) dmma_884(c[i][j][0], c[i][j][1], a[i], b[j]);
        }
        if (ch + 1 < chunks) stage(buf ^ 1);
        __syncthreads();
    }
    // accumulator fragment: lane holds rows lane/4, columns 2 (lane%4) + {0, 1} of each 8 x 8 block
    tr = 0.0;
    dev = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int gi = bi + wm + i * 8 + fr, gj = bj + wn + j * 8 + 2 * fk;
            if (gi >= d) continue;
            double v0 = alpha * c[i][j][0], v1 = alpha * c[i][j][1];
            if (gi == gj) { v0 += beta_diag; tr += v0; }
            if (gi == gj + 1) { v1 += beta_diag; tr += v1; }
            double* dst = C + (size_t)gi * d + gj;
            if (vec) {
                if (gj < d) *reinterpret_cast<double2*>(dst) = make_double2(v0, v1);
            } else {
                if (gj < d) dst[0] = v0;
                if (gj + 1 < d) dst[1] = v1;
            }
            if (gj < d) dev = fmaxf(dev, (float)fabs(v0 - (gi == gj ? 1.0 : 0.0)));
            if (gj + 1 < d) dev = fmaxf(dev, (float)fabs(v1 - (gi == gj + 1 ? 1.0 : 0.0)));
        }
}

// grid (ceil(d / 64), ceil(d / 64), problems)
__global__ void __launch_bounds__(256, 2)
dgemm_kernel(const DgemmBatch batch, int d)
{
    if (batch.dev_in != nullptr && *batch.dev_in < batch.tol) return;      // already converged
    if (batch.dev_clear != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 0)
        *batch.dev_clear = 0.0f;
    const DgemmProblem pr = blockIdx.z ? batch.p[1] : batch.p[0];   // no dynamically indexed copy of the parameter block
    float dev;
    double tr;
    dgemm_tile(pr.A, pr.B, pr.C, d, pr.alpha, pr.beta_diag, dev, tr);
    if (batch.dev_out != nullptr) {
        for (int o = 16; o > 0; o >>= 1) dev = fmaxf(dev, __shfl_xor_sync(0xffffffffu, dev, o));
        if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(batch.dev_out), __float_as_uint(dev));
    }
    if (pr.trace_out != nullptr && blockIdx.x == blockIdx.y) {
        // tiles that meet the diagonal only; reduce inside the block, one atomic per block
        __shared__ double red[256];
        red[threadIdx.x] = tr;
        __syncthreads();
        for (int s = 128; s > 0; s >>= 1) {
            if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
            __syncthreads();
        }
        if (threadIdx.x == 0) atomicAdd(pr.trace_out, red[0]);
    }
}

// out[0] = tr A      (single block)
__global__ void trace_kernel(const double* __restrict__ A, int d, double* __restrict__ out)
{
    __shared__ double r[256];
    double t = 0.0;
    for (int i = threadIdx.x; i < d; i += 256) t += A[(size_t)i * d + i];
    r[threadIdx.x] = t;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) r[threadIdx.x] += r[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) out[0] = r[0];
}

// scal[0] = |A|_F, scal[1] = tr A     (single block of 1024 threads: fixed summation order)
__global__ void __launch_bounds__(1024) norm_trace_kernel(const double* __restrict__ A, int d, double* __restrict__ scal)
{
    __shared__ double r1[1024], r2[1024];
    double s0 = 0.0, s1 = 0.0, t = 0.0;
    const size_t total = (size_t)d * d;
    size_t e = threadIdx.x;
    for (; e + 1024 < total; e += 2048) {                      // two independent chains per thread
        const double v0 = A[e], v1 = A[e + 1024];
        s0 += v0 * v0; s1 += v1 * v1;
    }
    if (e < total) { const double v = A[e]; s0 += v * v; }
    for (int i = threadIdx.x; i < d; i += 1024) t += A[(size_t)i * d + i];
    r1[threadIdx.x] = s0 + s1; r2[threadIdx.x] = t;
    __syncthreads();
    for (int k = 512; k > 0; k >>= 1) {
        if (threadIdx.x < k) { r1[threadIdx.x] += r1[threadIdx.x + k]; r2[threadIdx.x] += r2[threadIdx.x + k]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { scal[0] = sqrt(r1[0]); scal[1] = r2[0]; }
}

// Rank-deficient covariances (n < d) have eigenvalues that are zero up to roundoff, i.e. possibly
// slightly NEGATIVE, and Newton-Schulz diverges on a negative eigenvalue.  The iteration therefore
// runs on An + kNsDelta I (An = A/|A|_F), and the trace is corrected analytically:
//   tr sqrt(An) ~= tr Y - kNsDelta tr Z,      Y -> (An + dI)^(1/2),  Z -> (An + dI)^(-1/2)
// which is exact for null directions (sqrt(d) - d/sqrt(d) = 0) and O(d) ~ 1e-13 elsewhere.
constexpr double kNsDelta = 1e-13;

// Y = (A + A^T) / (2 |A|_F) + delta I, Z = I      (|A|_F read from scal[0])
__global__ void ns_init_kernel(const double* __restrict__ A, int d, const double* __restrict__ scal,
                               double* __restrict__ Y, double* __restrict__ Z)
{
    const double nrm = scal[0];
    const double inv = nrm > 0.0 ? 1.0 / nrm : 0.0;
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)d * d;
         e += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(e / d), j = (int)(e % d);
        Y[e] = 0.5 * (A[e] + A[(size_t)j * d + i]) * inv + ((i == j) ? kNsDelta : 0.0);
        Z[e] = (i == j) ? 1.0 : 0.0;
    }
}

// S = sqrt(|A|_F) * Y        (un-normalise a converged square root)
__global__ void ns_unscale_kernel(const double* __restrict__ Y, int d, const double* __restrict__ scal,
                                  double* __restrict__ S)
{
    const double f = sqrt(scal[0]);
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)d * d;
         e += (size_t)gridDim.x * blockDim.x) S[e] = f * Y[e];
}

// out[0] = fad, out[1] = tr sqrt(C1 C2), out[2] = relative residual |Y^2 - M/|M|_F|_F,
// out[3] = iterations, out[4] = |mu1-mu2|^2, out[5] = tr C1, out[6] = tr C2
__global__ void frechet_assemble_kernel(const double* __restrict__ mu1, const double* __restrict__ mu2, int d,
                                        const double* __restrict__ scalA /*|C1|_F, trC1*/,
                                        const double* __restrict__ trC2,
                                        const double* __restrict__ scalM /*|M|_F, trM*/,
                                        const double* __restrict__ trY, const double* __restrict__ trZ,
                                        const double* __restrict__ resid,
                                        int iters, double* __restrict__ out)
{
    __shared__ double red[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < d; i += 256) { const double df = mu1[i] - mu2[i]; s += df * df; }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const double tr_sqrt = sqrt(scalM[0]) * (trY[0] - kNsDelta * trZ[0]);
        out[0] = red[0] + scalA[1] + trC2[1] - 2.0 * tr_sqrt;
        out[1] = tr_sqrt;
        out[2] = resid ? sqrt(resid[0]) : 0.0;
        out[3] = (double)iters;
        out[4] = red[0];
        out[5] = scalA[1];
        out[6] = trC2[1];
    }
}

// resid[0] = | Y Y - Mn |_F^2 where Mn = sym(M)/|M|_F : computed as a fused GEMM epilogue would
// be overkill here; one extra GEMM into T then this reduction.
__global__ void resid_kernel(const double* __restrict__ YY, const double* __restrict__ M, int d,
                             const double* __restrict__ scalM, double* __restrict__ resid)
{
    __shared__ double red[256];
    const double inv = scalM[0] > 0.0 ? 1.0 / scalM[0] : 0.0;
    double s = 0.0;
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)d * d;
         e += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(e / d), j = (int)(e % d);
        const double m = 0.5 * (M[e] + M[(size_t)j * d + i]) * inv + ((i == j) ? kNsDelta : 0.0);
        const double r = YY[e] - m;
        s += r * r;
    }
    red[threadIdx.x] = s;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) red[threadIdx.x] += red[threadIdx.x + k];
        __syncthreads();
    }
    if (threadIdx.x == 0) atomicAdd(resid, red[0]);
}

}  // namespace fad
