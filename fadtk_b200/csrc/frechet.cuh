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
// One chain serves every entry point: item z of a group owns the z-th d x d matrix of each operand, every stage
// is one launch over all items, and each item carries its own convergence flags.  The single-problem entry points
// run it with one item; fad_frechet_batched scores many eval sets (songs) against one baseline in lock-step,
// M_z = S C_z S with S = C_base^(1/2) cached.
// All scalars (norms, traces) stay on the device; the chain is launched without host syncs.
#pragma once
#include <stdint.h>

#include "sm90.cuh"

namespace fad {

// One 64 x 64 tile of C = alpha A B + beta_diag I per 256-thread CTA on the FP64 TENSOR pipe
// (mma.sync m8n8k4 f64 -> SASS DMMA.8x8x4, the fp64 MMA shape of sm_90a; wgmma has no f64 kind).
// Returns max |C - I| over this thread's outputs.
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

__device__ __forceinline__ void dgemm_tile(const double* __restrict__ A, const double* __restrict__ B,
                                           double* __restrict__ C, int d, double alpha, double beta_diag,
                                           float& dev)
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
                for (int j = 0; j < 2; ++j) sm90::dmma_884(c[i][j][0], c[i][j][1], a[i], b[j]);
        }
        if (ch + 1 < chunks) stage(buf ^ 1);
        __syncthreads();
    }
    // accumulator fragment: lane holds rows lane/4, columns 2 (lane%4) + {0, 1} of each 8 x 8 block
    dev = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int gi = bi + wm + i * 8 + fr, gj = bj + wn + j * 8 + 2 * fk;
            if (gi >= d) continue;
            double v0 = alpha * c[i][j][0], v1 = alpha * c[i][j][1];
            if (gi == gj) v0 += beta_diag;
            if (gi == gj + 1) v1 += beta_diag;
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

// C_z = alpha A_z B_z + beta_diag I for two strided families of problems in one launch:
// grid (ceil(d / 64), ceil(d / 64), families * items), blockIdx.z = item + family * items.  A stride of 0 shares the
// operand between items (the cached baseline root).
// Convergence control without host round trips: flags holds three rotating float slots of max |W - I| per item.  A
// launch whose in_slot (the previous iteration) is below tol returns at once for that item, so a fixed-length launch
// sequence costs only launch latency once an item has converged; out_slot receives max |C - I| (float bits,
// atomicMax), clear_slot is zeroed for a later iteration.  Slot -1 or null flags = unused.
struct DgemmFamily { const double* A; const double* B; double* C; long long sA, sB, sC; double alpha, beta_diag; };
struct DgemmStrided {
    DgemmFamily f[2];
    int items;
    float* flags;          // [items][3] or null
    int in_slot, out_slot, clear_slot;
    float tol;
};

__global__ void __launch_bounds__(256, 2)
dgemm_strided_kernel(const DgemmStrided p, int d)
{
    const int fam = blockIdx.z >= p.items ? 1 : 0;
    const int z = blockIdx.z - fam * p.items;
    float* fl = p.flags ? p.flags + (size_t)z * 3 : nullptr;
    if (fl && p.in_slot >= 0 && fl[p.in_slot] < p.tol) return;             // this item has converged
    if (fl && p.clear_slot >= 0 && fam == 0 && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) fl[p.clear_slot] = 0.0f;
    const DgemmFamily f = fam ? p.f[1] : p.f[0];                          // no dynamically indexed copy of the parameter block
    float dev;
    dgemm_tile(f.A + (size_t)z * f.sA, f.B + (size_t)z * f.sB, f.C + (size_t)z * f.sC, d, f.alpha, f.beta_diag, dev);
    if (fl && p.out_slot >= 0) {
        for (int o = 16; o > 0; o >>= 1) dev = fmaxf(dev, __shfl_xor_sync(0xffffffffu, dev, o));
        if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned int*>(fl + p.out_slot), __float_as_uint(dev));
    }
}

// scal[z] = {|A_z|_F, tr A_z}; one block of 1024 threads per item, fixed summation order
__global__ void __launch_bounds__(1024) norm_trace_kernel(const double* __restrict__ A, int d, double* __restrict__ scal /*[items][2]*/)
{
    __shared__ double r1[1024], r2[1024];
    const double* Az = A + (size_t)blockIdx.x * d * d;
    double s0 = 0.0, s1 = 0.0, t = 0.0;
    const size_t total = (size_t)d * d;
    size_t e = threadIdx.x;
    for (; e + 1024 < total; e += 2048) {                      // two independent chains per thread
        const double v0 = Az[e], v1 = Az[e + 1024];
        s0 += v0 * v0; s1 += v1 * v1;
    }
    if (e < total) { const double v = Az[e]; s0 += v * v; }
    for (int i = threadIdx.x; i < d; i += 1024) t += Az[(size_t)i * d + i];
    r1[threadIdx.x] = s0 + s1; r2[threadIdx.x] = t;
    __syncthreads();
    for (int k = 512; k > 0; k >>= 1) {
        if (threadIdx.x < k) { r1[threadIdx.x] += r1[threadIdx.x + k]; r2[threadIdx.x] += r2[threadIdx.x + k]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { scal[2 * blockIdx.x] = sqrt(r1[0]); scal[2 * blockIdx.x + 1] = r2[0]; }
}

// Rank-deficient covariances (n < d) have eigenvalues that are zero up to roundoff, i.e. possibly
// slightly NEGATIVE, and Newton-Schulz diverges on a negative eigenvalue.  The iteration therefore
// runs on An + kNsDelta I (An = A/|A|_F), and the trace is corrected analytically:
//   tr sqrt(An) ~= tr Y - kNsDelta tr Z,      Y -> (An + dI)^(1/2),  Z -> (An + dI)^(-1/2)
// which is exact for null directions (sqrt(d) - d/sqrt(d) = 0) and O(d) ~ 1e-13 elsewhere.
constexpr double kNsDelta = 1e-13;

// Y_z = sym(A_z)/|A_z|_F + delta I, Z_z = I, flags_z = {0, 0, 1e30} (slot (k-1)%3 for k = 0 is slot 2);
// |A_z|_F read from scal[2z].  grid (blocks, items)
__global__ void __launch_bounds__(256)
ns_init_kernel(const double* __restrict__ A, int d, const double* __restrict__ scal,
               double* __restrict__ Y, double* __restrict__ Z, float* __restrict__ flags)
{
    const int z = blockIdx.y;
    const double nrm = scal[2 * z];
    const double inv = nrm > 0.0 ? 1.0 / nrm : 0.0;
    const double* Az = A + (size_t)z * d * d;
    double* Yz = Y + (size_t)z * d * d;
    double* Zz = Z + (size_t)z * d * d;
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)d * d; e += (size_t)gridDim.x * blockDim.x) {
        const int i = (int)(e / d), j = (int)(e % d);
        Yz[e] = 0.5 * (Az[e] + Az[(size_t)j * d + i]) * inv + ((i == j) ? kNsDelta : 0.0);
        Zz[e] = (i == j) ? 1.0 : 0.0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { flags[3 * z] = 0.0f; flags[3 * z + 1] = 0.0f; flags[3 * z + 2] = 1.0e30f; }
}

// S = sqrt(|A|_F) * Y        (un-normalise a converged square root)
__global__ void ns_unscale_kernel(const double* __restrict__ Y, int d, const double* __restrict__ scal,
                                  double* __restrict__ S)
{
    const double f = sqrt(scal[0]);
    for (size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x; e < (size_t)d * d;
         e += (size_t)gridDim.x * blockDim.x) S[e] = f * Y[e];
}

// out[z][0] = fad, [1] = tr sqrt(C1 C2_z), [2] = relative residual |Y^2 - M/|M|_F|_F (0 without resid),
// [3] = iterations, [4] = |mu1-mu2_z|^2, [5] = tr C1, [6] = tr C2_z, [7] = row count (left alone without offsets).
// An item with ok[z] == 0 gets NaN in [0], [1]; null ok = every item is good.  One block per item.
__global__ void __launch_bounds__(256)
frechet_assemble_kernel(const double* __restrict__ mu1, const double* __restrict__ mu2 /*[items][d]*/, int d,
                        const double* __restrict__ scal1 /*|C1|_F, tr C1*/,
                        const double* __restrict__ scalC /*[items][2]: |C2_z|_F, tr C2_z*/,
                        const double* __restrict__ scalM /*[items][2]*/,
                        const double* __restrict__ Y, const double* __restrict__ Z, const double* __restrict__ resid,
                        const int* __restrict__ ok, const long long* __restrict__ offsets,
                        int iters, double* __restrict__ out)
{
    __shared__ double r0[256], r1[256], r2[256];
    const int z = blockIdx.x;
    const double* Yz = Y + (size_t)z * d * d;
    const double* Zz = Z + (size_t)z * d * d;
    double s = 0.0, ty = 0.0, tz = 0.0;
    for (int i = threadIdx.x; i < d; i += 256) {
        const double df = mu1[i] - mu2[(size_t)z * d + i];
        s += df * df;
        ty += Yz[(size_t)i * d + i];
        tz += Zz[(size_t)i * d + i];
    }
    r0[threadIdx.x] = s; r1[threadIdx.x] = ty; r2[threadIdx.x] = tz;
    __syncthreads();
    for (int k = 128; k > 0; k >>= 1) {
        if (threadIdx.x < k) { r0[threadIdx.x] += r0[threadIdx.x + k]; r1[threadIdx.x] += r1[threadIdx.x + k]; r2[threadIdx.x] += r2[threadIdx.x + k]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        double* o = out + (size_t)z * 8;
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        const double tr_sqrt = sqrt(scalM[2 * z]) * (r1[0] - kNsDelta * r2[0]);
        const bool good = ok == nullptr || ok[z] != 0;
        o[0] = good ? r0[0] + scal1[1] + scalC[2 * z + 1] - 2.0 * tr_sqrt : nan;
        o[1] = good ? tr_sqrt : nan;
        o[2] = resid ? sqrt(resid[0]) : 0.0;
        o[3] = (double)iters;
        o[4] = r0[0];
        o[5] = scal1[1];
        o[6] = scalC[2 * z + 1];
        if (offsets) o[7] = (double)(offsets[z + 1] - offsets[z]);
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
