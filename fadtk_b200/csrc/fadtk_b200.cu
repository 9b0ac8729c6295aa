// Host side of the C ABI declared in include/fadtk_b200.h: owns device weights and workspaces,
// encodes TMA descriptors, launches the sm_90a kernels.  No torch, no CUTLASS.
#include "../../include/fadtk_b200.h"

#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cxxabi.h>
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <initializer_list>
#include <memory>
#include <set>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "conv_gemm.cuh"
#include "frontend.cuh"
#include "stats.cuh"
#include "frechet.cuh"
#include "clap.cuh"
#include "resample.cuh"
#include "whisper.cuh"
#include "encodec.cuh"
#include "wav2vec.cuh"
#include "attention_wgmma.cuh"
#include "kad.cuh"
#include "prdc.cuh"

namespace {

thread_local std::string g_err;

int fail(const std::string& m) { g_err = m; return 1; }

#define CK(call)                                                                          \
    do {                                                                                  \
        cudaError_t e_ = (call);                                                          \
        if (e_ != cudaSuccess)                                                            \
            return fail(std::string(#call) + ": " + cudaGetErrorString(e_));              \
    } while (0)

// The one owner of device memory in the library: a block of at least size() bytes, freed by the destructor.
class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(DeviceBuffer&& o) noexcept : p_(o.p_), bytes_(o.bytes_) { o.p_ = nullptr; o.bytes_ = 0; }  // no copies
    ~DeviceBuffer() { if (p_) cudaFree(p_); }

    // at least `bytes`: reallocates only when the block is smaller, and does not keep its contents
    int grow(size_t bytes) {
        if (bytes_ >= bytes) return 0;
        if (p_) cudaFree(p_);
        p_ = nullptr; bytes_ = 0;
        CK(cudaMalloc(&p_, bytes));
        bytes_ = bytes;
        return 0;
    }
    template <typename T = void> T* get() const { return static_cast<T*>(p_); }
    size_t size() const { return bytes_; }

private:
    void* p_ = nullptr;
    size_t bytes_ = 0;
};

// The weights and fixed workspaces of a loaded model live in a std::vector<DeviceBuffer> of its state; the typed
// pointers of the state are views into it.  A copy of `bytes` host bytes at *dst:
template <typename T>
int upload(std::vector<DeviceBuffer>& mem, T** dst, const void* src, size_t bytes) {
    DeviceBuffer b;
    if (b.grow(bytes)) return 1;
    CK(cudaMemcpy(b.get(), src, bytes, cudaMemcpyHostToDevice));
    *dst = b.get<T>();
    mem.push_back(std::move(b));
    return 0;
}
// `bytes` uninitialised (or zeroed) bytes at *dst
template <typename T>
int alloc(std::vector<DeviceBuffer>& mem, T** dst, size_t bytes, bool zero = false) {
    DeviceBuffer b;
    if (b.grow(bytes)) return 1;
    if (zero) CK(cudaMemset(b.get(), 0, bytes));
    *dst = b.get<T>();
    mem.push_back(std::move(b));
    return 0;
}

// One buffer of a workspace: n elements of T (rounded up to 256 bytes), whose address carve() stores in p
template <typename T> struct Slot { T** p; size_t bytes; };
template <typename T> Slot<T> slot(T*& p, size_t n) { return {&p, (n * sizeof(T) + 255) & ~size_t(255)}; }

// A workspace laid out in buf: the slots in the order given.  Grows buf to the total and points every slot at its place.
template <typename... T>
int carve(DeviceBuffer& buf, Slot<T>... s) {
    if (buf.grow((s.bytes + ... + size_t(0)))) return 1;
    unsigned char* q = buf.get<unsigned char>();
    ((*s.p = reinterpret_cast<T*>(q), q += s.bytes), ...);
    return 0;
}

// A load checks every tensor pointer before it touches its model's slot.
int check_tensors(const char* fn, const void* const* t, int n_tensors) {
    for (int i = 0; i < n_tensors; ++i)
        if (!t[i]) return fail(std::string(fn) + ": null tensor pointer");
    return 0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// fp16 tensor, innermost dimension first; 128-B swizzle, zero fill out of bounds.
int encode_f16_map(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                   const uint64_t* strides_bytes /*rank-1*/, const uint32_t* box) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return fail("cuTensorMapEncodeTiled entry point not available");
    cuuint64_t gdim[5], gstr[4];
    cuuint32_t bdim[5], estr[5];
    for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = 1; }
    for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base),
                    gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        char buf[256];
        snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d) rank=%d dims=%llu,%llu box=%u,%u", (int)r, rank,
                 (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0), box[0], rank > 1 ? box[1] : 0);
        return fail(buf);
    }
    return 0;
}

struct LayerGeom {
    int taps, Cin, Cout, H, W, relu, pool;
    int box_w, box_h, box_n, n_tile;
    int split_w;      // 0: fp16 weights; 1: fp16 hi/lo pair (interleaved per 128-row tile), two fp16 MMAs
};

int make_geom(LayerGeom& g, int H, int W, int Cin, int Cout, int taps, int relu, int pool, int split_w) {
    g.taps = taps; g.Cin = Cin; g.Cout = Cout; g.H = H; g.W = W; g.relu = relu; g.pool = pool;
    g.split_w = split_w;
    if (Cin % 64 != 0) return fail("Cin must be a multiple of 64");
    if (taps != 1 && taps != 9) return fail("taps must be 1 or 9");
    if (H == 1 && W == 1) { g.box_w = 1; g.box_h = 1; g.box_n = 128; }
    else {
        g.box_w = W < 16 ? W : 16;
        if (g.box_w != 8 && g.box_w != 16) return fail("W must be 8 or a multiple of 16");
        if (W % g.box_w != 0) return fail("W must be a multiple of the 16-pixel box");
        int bh = 1;
        while (bh * 2 <= 128 / g.box_w && H % (bh * 2) == 0) bh *= 2;
        g.box_h = bh;
        g.box_n = 128 / (g.box_w * g.box_h);
    }
    if (pool && (g.box_h % 2 != 0 || g.box_w % 2 != 0)) return fail("pooling needs even tile boxes");
    if (Cout % 128 != 0) return fail("Cout must be a multiple of 128");
    g.n_tile = 128;                          // one m64n128 wgmma accumulator per consumer warpgroup
    return 0;
}

// the loaded models, one slot each: set by a load that succeeded, empty after one that failed part way
struct VggState;       // below
struct ClapState;      // clap_host.inc
struct WhisperState;   // whisper_host.inc
struct EncodecState;   // encodec_host.inc
struct W2vState;       // wav2vec_host.inc

}  // namespace

struct fad_handle {
    int device = 0;
    int num_sms = 0;
    int max_examples = 0;
    long long launches = 0;          // kernels launched through `launch` (fad_launch_count)
    int gemm_clusters[2] = {};       // co-resident CTA pairs of the wgmma GEMM, by weight mode (fad_create)

    // front-end tables
    std::vector<DeviceBuffer> mem;
    double *d_twiddle = nullptr, *d_hann = nullptr, *d_melw = nullptr;
    int *d_mel_start = nullptr, *d_mel_count = nullptr;

    // workspaces, grown on demand
    DeviceBuffer ws_tiles, ws_sums, gather_buf;     // statistics
    DeviceBuffer fr_buf;                            // Frechet (FrechetWorkspace)
    DeviceBuffer rs_bank, rs_mono;                  // resampler filter bank and mono mix
    int rs_in = 0, rs_out = 0;                      // the rate pair of rs_bank
    DeviceBuffer pair_buf;                          // fad_kad_*, fad_knn_radii_sq, fad_prdc_counts, fad_realism, fad_nearest (pair_prepare)
    DeviceBuffer agree_buf;                         // the sharded entries: the ranks' argument descriptor (agree)
    // hi/lo weight tensors whose lo parts are all zero, by address (note_split_weights).  Every hi/lo tensor is noted
    // at its current address before any GEMM reads it: upload_split and fad_vggish_load note each one they upload,
    // fad_umma_layer and fad_linear the caller's on every call.  An entry left behind for a freed address is
    // therefore overwritten before it can be read.
    std::set<const void*> zero_lo;

    void* nccl_comm = nullptr;   // ncclComm_t created by fad_comm_init (NCCL is dlopen'ed, never linked)

    std::unique_ptr<VggState> vgg;
    std::unique_ptr<ClapState> clap;
    std::unique_ptr<WhisperState> whisper;
    std::unique_ptr<EncodecState> encodec;
    std::unique_ptr<W2vState> w2v;
    ~fad_handle();      // at the end of the file, where the state types are complete

    // optional per-category timing with CUDA events recorded on the launching stream
    bool prof_on = false;
    std::vector<cudaEvent_t> ev_pool;
    size_t ev_used = 0;
    struct Span { int cat; size_t e0, e1; };
    std::vector<Span> spans;
    double prof_ms[FAD_PROF_CATEGORIES] = {};
    long long prof_count[FAD_PROF_CATEGORIES] = {};
};

namespace {

// The kernel's demangled signature, for error messages.
std::string kernel_name(const void* kernel) {
    const char* mangled = nullptr;
    if (cudaFuncGetName(&mangled, kernel) != cudaSuccess || !mangled) return "kernel launch";
    int status = 0;
    char* demangled = abi::__cxa_demangle(mangled, nullptr, nullptr, &status);
    const std::string name = demangled ? demangled : mangled;
    free(demangled);
    return name;
}

// Every kernel launch of the library: kernel<<<grid, block, smem, st>>>(args...) with the launch attributes
// attrs[0, n_attrs), counted in h->launches.  A grid with a zero dimension launches and counts nothing.  The arguments
// are converted to the kernel's parameter types, and defaulted parameters must be passed too.
template <typename... Params, typename... Args>
int launch_attrs(fad_handle* h, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                 cudaLaunchAttribute* attrs, unsigned n_attrs, Args&&... args) {
    if (grid.x == 0 || grid.y == 0 || grid.z == 0) return 0;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cfg.attrs = attrs;
    cfg.numAttrs = n_attrs;
    cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
    const cudaError_t last = cudaGetLastError();     // also clears the error state a failed launch leaves behind
    if (e == cudaSuccess) e = last;
    if (e != cudaSuccess) return fail(kernel_name((const void*)kernel) + ": " + cudaGetErrorString(e));
    h->launches++;
    return 0;
}
template <typename... Params, typename... Args>
int launch(fad_handle* h, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    return launch_attrs(h, kernel, grid, block, smem, st, nullptr, 0, std::forward<Args>(args)...);
}

// The wgmma GEMM (conv_gemm.cuh) by weight mode, 0: fp16, 1: fp16 hi/lo pair.  Stages: as many 32 / 48 KiB stages as
// fit next to the two 32 KiB epilogue tiles in 227 KiB.
template <int WMODE> struct Gemm {
    static constexpr int kStages = WMODE ? 3 : 4;
    static constexpr uint32_t kSmem = fad::conv_gemm_smem_bytes<128, kStages, WMODE>();
    static_assert(kSmem <= 227 * 1024, "over the per-CTA shared-memory limit");
    static constexpr auto kernel = fad::conv_gemm_kernel<128, kStages, WMODE>;
};

cudaLaunchAttribute cta_pair() {
    cudaLaunchAttribute attr = {};
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = fad::kClusterCtas; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    return attr;
}

// Shared memory above the default for the GEMM, and how many of its CTA pairs fit on the device at once.
template <int WMODE>
int setup_gemm(fad_handle* h) {
    CK(cudaFuncSetAttribute(Gemm<WMODE>::kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Gemm<WMODE>::kSmem));
    cudaLaunchAttribute attr = cta_pair();
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(fad::kClusterCtas * (unsigned)h->num_sms);
    cfg.blockDim = dim3(fad::kConvGemmThreads);
    cfg.dynamicSmemBytes = Gemm<WMODE>::kSmem;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    CK(cudaOccupancyMaxActiveClusters(&h->gemm_clusters[WMODE], Gemm<WMODE>::kernel, &cfg));
    if (h->gemm_clusters[WMODE] <= 0) return fail("conv_gemm_kernel: no CTA pair fits on the device");
    return 0;
}

template <int WMODE>
int launch_conv_gemm(fad_handle* h, const CUtensorMap& mx, const CUtensorMap& mw, const fad::ConvGemmParams& p, cudaStream_t st) {
    const int units = (p.img_groups * p.tiles_h * p.tiles_w + 1) / 2 * p.n_tiles;
    cudaLaunchAttribute attr = cta_pair();
    return launch_attrs(h, Gemm<WMODE>::kernel, dim3(fad::kClusterCtas * (unsigned)std::min(units, h->gemm_clusters[WMODE])),
                        dim3(fad::kConvGemmThreads), Gemm<WMODE>::kSmem, st, &attr, 1, mx, mw, p);
}

// a_cols: channels actually stored per pixel/row of the activation (<= g.Cin); the TMA box reads
// zeros beyond it, so a K that is not a multiple of 64 needs no padding columns in HBM.
int encode_layer_maps(const LayerGeom& g, const void* x, long long nb_dim, const void* w,
                      CUtensorMap* mx, CUtensorMap* mw, int a_cols = 0, long long a_row_stride = 0) {
    const uint64_t ac = a_cols > 0 ? (uint64_t)a_cols : (uint64_t)g.Cin;
    const uint64_t xd[4] = {ac, (uint64_t)g.W, (uint64_t)g.H, (uint64_t)nb_dim};
    uint64_t xs[3] = {ac * 2, (uint64_t)g.W * ac * 2, (uint64_t)g.H * g.W * ac * 2};
    // 1x1 geometry only: rows a_row_stride elements apart (< a_cols = overlapping rows, e.g. the sliding
    // windows of a strided 1-D convolution read straight from the [T][C] activation, no im2col copy)
    if (a_row_stride > 0) xs[0] = xs[1] = xs[2] = (uint64_t)a_row_stride * 2;
    const uint32_t xb[4] = {64, (uint32_t)g.box_w, (uint32_t)g.box_h, (uint32_t)g.box_n};
    if (encode_f16_map(mx, x, 4, xd, xs, xb)) return 1;
    const uint64_t K = (uint64_t)g.taps * g.Cin;
    const uint64_t rows_mul = g.split_w ? 2 : 1;
    const uint64_t wd[2] = {K, (uint64_t)g.Cout * rows_mul};
    const uint64_t ws[1] = {K * 2};
    // rows per weight box: each CTA of a pair fetches half of a tile's rows (split: the hi or the lo rows) for both
    const uint32_t wb[2] = {64, (uint32_t)(g.n_tile * rows_mul / fad::kClusterCtas)};
    return encode_f16_map(mw, w, 2, wd, ws, wb);
}

// Encoder self-attention on wgmma (attention_wgmma.cuh).  qkv: fp16 [clips * S][3 d] (q | k | v, head h at column h * 64),
// out: fp16 [clips * S][d].
int launch_attention_wgmma(fad_handle* h, const __half* qkv, long long n_clips, int S, int d, int heads, __half* out, cudaStream_t st) {
    if (heads * 64 != d) return fail("attention_wgmma: head dimension must be 64");
    CUtensorMap map;
    const uint64_t dims[3] = {(uint64_t)3 * d, (uint64_t)S, (uint64_t)n_clips};
    const uint64_t strides[2] = {(uint64_t)3 * d * 2, (uint64_t)S * 3 * d * 2};
    const uint32_t box[3] = {64, 128, 1};
    if (encode_f16_map(&map, qkv, 3, dims, strides, box)) return 1;
    fad::AttnParams p;
    p.S = S; p.d = d; p.heads = heads; p.out = out;
    return launch(h, fad::attention_wgmma_kernel, dim3((S + 127) / 128, heads, (unsigned)n_clips), fad::kAtThreads, fad::kAtSmem,
                  st, map, p);
}

int run_layer(fad_handle* h, const LayerGeom& g, const CUtensorMap& mx, const CUtensorMap& mw, const void* w,
              int NB, const float* bias, void* out, float* out_f32, cudaStream_t st,
              float* resid = nullptr, int resid_C = 0, int resid_res = 0, int resid_shift = 0, int n_valid = 0) {
    fad::ConvGemmParams p;
    p.taps = g.taps; p.cblks = g.Cin / 64;
    p.box_w = g.box_w; p.box_h = g.box_h; p.box_n = g.box_n;
    p.tiles_w = g.W / g.box_w; p.tiles_h = g.H / g.box_h;
    p.img_groups = (NB + g.box_n - 1) / g.box_n;
    p.n_tiles = g.Cout / g.n_tile;
    p.H = g.H; p.W = g.W; p.NB = NB; p.Cout = g.Cout;
    p.n_valid = n_valid > 0 ? n_valid : g.Cout;
    p.ld_out = p.n_valid;
    p.relu = g.relu; p.pool = g.pool;
    p.bias = bias; p.out = reinterpret_cast<__half*>(out); p.out_f32 = out_f32;
    p.resid = resid; p.resid_C = resid_C; p.resid_res = resid_res; p.resid_shift = resid_shift;
    p.lo_adds = g.split_w == 1 && h->zero_lo.count(w) == 0;
    if (g.split_w) return launch_conv_gemm<1>(h, mx, mw, p, st);
    return launch_conv_gemm<0>(h, mx, mw, p, st);
}

// max |Wl| over the lo parts of a packed hi/lo weight tensor ([hi: 128 rows | lo: 128 rows] per tile), as float bits
__global__ void wlo_absmax_kernel(const __half* __restrict__ w, long long n_tiles, long long K, unsigned int* __restrict__ out) {
    float m = 0.f;
    const long long total = n_tiles * 128 * K;
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const long long row = e / K, k = e - row * K;
        const long long t = row >> 7, j = row & 127;
        m = fmaxf(m, fabsf(__half2float(w[((t * 256 + 128 + j) * K) + k])));
    }
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}
// Whether the lo parts of a hi/lo weight tensor ([2 * 128 * n_tiles, K], device) are all zero, as they are for weights
// that are exact in fp16.  Their lo wgmmas then add exact zeros, which do not truncate the accumulator, and the GEMM's
// unshrink counts the hi products only (ConvGemmParams::lo_adds).  Every hi/lo tensor is noted when it is uploaded;
// the caller's tensors (the stage entries) on every call.  Synchronous.
int note_split_weights(fad_handle* h, const void* w, long long n_tiles, long long K, cudaStream_t st) {
    DeviceBuffer d_max;
    if (d_max.grow(4)) return 1;
    unsigned int mx = 0;
    const unsigned blocks = (unsigned)std::max<long long>(1, std::min<long long>((n_tiles * 128 * K + 255) / 256, (long long)h->num_sms * 16));
    CK(cudaMemsetAsync(d_max.get(), 0, 4, st));
    if (launch(h, wlo_absmax_kernel, blocks, 256, 0, st, reinterpret_cast<const __half*>(w), n_tiles, K, d_max.get<unsigned int>()))
        return 1;
    CK(cudaMemcpyAsync(&mx, d_max.get(), 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (mx == 0) h->zero_lo.insert(w); else h->zero_lo.erase(w);
    return 0;
}

// an fp16 hi/lo weight tensor [2 n, k] (n a multiple of 128), noted for the GEMM's truncation compensation
int upload_split(fad_handle* h, std::vector<DeviceBuffer>& mem, __half** dst, const void* src, size_t n, size_t k) {
    if (upload(mem, dst, src, 2 * n * k * 2)) return 1;
    return note_split_weights(h, *dst, (long long)(n / 128), (long long)k, 0);
}

// VGGish layer table: H, W are the conv's spatial size (input == un-pooled output)
struct VggLayer { int H, W, Cin, Cout, taps, relu, pool; };
const VggLayer kVgg[8] = {
    {48, 32, 64, 128, 9, 1, 1},     // conv2  -> [24,16,128]
    {24, 16, 128, 256, 9, 1, 0},    // conv3_1
    {24, 16, 256, 256, 9, 1, 1},    // conv3_2 -> [12,8,256]
    {12, 8, 256, 512, 9, 1, 0},     // conv4_1
    {12, 8, 512, 512, 9, 1, 1},     // conv4_2 -> [6,4,512] == [12288]
    {1, 1, 12288, 4096, 1, 1, 0},   // fc1
    {1, 1, 4096, 4096, 1, 1, 0},    // fc2
    {1, 1, 4096, 128, 1, 0, 0},     // fc3 (no ReLU: fadtk/model_loader.py:102-103)
};
// bytes of fp16 activation per example produced by: conv1, conv2, conv3_1, conv3_2, conv4_1, conv4_2, fc1, fc2
const size_t kActElems[8] = {48 * 32 * 64, 24 * 16 * 128, 24 * 16 * 256, 12 * 8 * 256,
                             12 * 8 * 512, 6 * 4 * 512, 4096, 4096};

struct VggState {
    std::vector<DeviceBuffer> mem;      // everything below points into it
    float *conv1_w = nullptr, *conv1_b = nullptr;
    __half* w[8] = {};         // the layers of kVgg: conv2 .. conv4_2, fc1 .. fc3
    float* b[8] = {};
    // activations, sized for max_examples
    float* logmel = nullptr;
    __half* act[8] = {};       // act[0]=conv1 out ... act[5]=conv6 out (flattened), act[6..7]=fc1, fc2 out
    // per-layer cached descriptors for the fixed pipeline
    CUtensorMap map_x[8], map_w[8];
    LayerGeom geom[8];
};

void build_frontend_tables(std::vector<double>& tw, std::vector<double>& hann,
                           std::vector<double>& melw, std::vector<int>& mstart, std::vector<int>& mcount) {
    const double PI = 3.14159265358979323846;
    tw.resize(512); hann.resize(fad::kWin);
    for (int k = 0; k < 256; ++k) {
        tw[2 * k] = std::cos(-2.0 * PI * k / 512.0);
        tw[2 * k + 1] = std::sin(-2.0 * PI * k / 512.0);
    }
    for (int n = 0; n < fad::kWin; ++n) hann[n] = 0.5 - 0.5 * std::cos(2.0 * PI / fad::kWin * n);
    // HTK mel filterbank, 64 bands over 125..7500 Hz on 257 bins of 0..8000 Hz; DC bin zeroed
    auto mel = [](double f) { return 1127.0 * std::log(1.0 + f / 700.0); };
    std::vector<double> bins(fad::kBins), edges(fad::kMel + 2);
    for (int i = 0; i < fad::kBins; ++i) bins[i] = mel(8000.0 * i / (fad::kBins - 1));
    const double lo = mel(125.0), hi = mel(7500.0);
    for (int i = 0; i < fad::kMel + 2; ++i) edges[i] = lo + (hi - lo) * i / (fad::kMel + 1);
    melw.assign(fad::kMel * fad::kMelMaxTaps, 0.0);
    mstart.assign(fad::kMel, 0); mcount.assign(fad::kMel, 0);
    for (int b = 0; b < fad::kMel; ++b) {
        const double l = edges[b], c = edges[b + 1], u = edges[b + 2];
        int first = -1, cnt = 0;
        for (int i = 1; i < fad::kBins; ++i) {            // bin 0 (DC) has zero weight
            const double w = std::fmax(0.0, std::fmin((bins[i] - l) / (c - l), (u - bins[i]) / (u - c)));
            if (w > 0.0) {
                if (first < 0) first = i;
                const int off = i - first;
                if (off < fad::kMelMaxTaps) { melw[b * fad::kMelMaxTaps + off] = w; cnt = off + 1; }
            }
        }
        mstart[b] = first < 0 ? 0 : first;
        mcount[b] = cnt;
    }
}

size_t prof_begin(fad_handle* h, cudaStream_t st) {
    if (!h->prof_on) return 0;
    if (h->ev_used == h->ev_pool.size()) { cudaEvent_t e; cudaEventCreate(&e); h->ev_pool.push_back(e); }
    cudaEventRecord(h->ev_pool[h->ev_used], st);
    return h->ev_used++;
}
void prof_end(fad_handle* h, int cat, size_t e0, cudaStream_t st) {
    if (!h->prof_on) return;
    const size_t e1 = prof_begin(h, st);
    h->spans.push_back({cat, e0, e1});
}

// Exact Gram statistics on the FP64 tensor pipe (stats.cuh): acc += the packed statistics of E [n_rows, d] - shift.
// In = __half (embeddings) or double (per-file mean rows, no shift).  Only the embedding statistics are profiled.
template <typename In>
int launch_stats_dmma(fad_handle* h, const In* E, long long n_rows, int d, const __half* shift, double* acc, cudaStream_t st) {
    constexpr bool kProf = sizeof(In) == 2;
    if (d <= 0 || d % 64 != 0) return fail("d must be a positive multiple of 64");
    fad::StatsDmmaParams p;
    p.n_rows = n_rows; p.d = d; p.n_tiles = d / fad::kSdTile;
    p.n_pairs = p.n_tiles * (p.n_tiles + 1) / 2;
    const long long stages = (n_rows + fad::kSdRows - 1) / fad::kSdRows;
    long long want = (4LL * h->num_sms + p.n_pairs - 1) / p.n_pairs;       // ~2 waves at 2 CTAs per SM
    if (want < 1) want = 1;
    long long per = (stages + want - 1) / want;                             // 16-row stages per split
    if (per < 4) per = 4;
    p.n_splits = (int)((stages + per - 1) / per);
    p.rows_per_split = per * fad::kSdRows;
    p.shift = shift;
    const size_t jobs = (size_t)p.n_pairs * p.n_splits;
    if (h->ws_tiles.grow(jobs * fad::kSdTile * fad::kSdTile * 8)) return 1;
    if (h->ws_sums.grow((size_t)p.n_tiles * p.n_splits * fad::kSdTile * 8)) return 1;
    p.ws_tiles = h->ws_tiles.get<double>(); p.ws_sums = h->ws_sums.get<double>();
    size_t ev = kProf ? prof_begin(h, st) : 0;
    if (launch(h, fad::stats_dmma_kernel<In>, (unsigned)jobs, 256, 0, st, E, p)) return 1;
    if (kProf) { prof_end(h, FAD_PROF_STATS, ev, st); ev = prof_begin(h, st); }
    if (launch(h, fad::stats_dmma_reduce_kernel, dim3(p.n_pairs, fad::kSdTile * fad::kSdTile / 256), 256, 0, st, p, acc)) return 1;
    if (kProf) prof_end(h, FAD_PROF_STATS_REDUCE, ev, st);
    return 0;
}

}  // namespace

extern "C" {

int fad_version(void) { return 1; }

int fad_profile_enable(fad_handle* h, int on) {
    if (!h) return fail("null handle");
    h->prof_on = on != 0;
    return 0;
}

int fad_profile_collect(fad_handle* h, double* ms_out, long long* count_out, int reset) {
    if (!h) return fail("null handle");
    CK(cudaSetDevice(h->device));
    CK(cudaDeviceSynchronize());
    for (const auto& sp : h->spans) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, h->ev_pool[sp.e0], h->ev_pool[sp.e1]) == cudaSuccess) {
            h->prof_ms[sp.cat] += ms; h->prof_count[sp.cat]++;
        }
    }
    h->spans.clear(); h->ev_used = 0;
    for (int i = 0; i < FAD_PROF_CATEGORIES; ++i) {
        if (ms_out) ms_out[i] = h->prof_ms[i];
        if (count_out) count_out[i] = h->prof_count[i];
        if (reset) { h->prof_ms[i] = 0.0; h->prof_count[i] = 0; }
    }
    return 0;
}
const char* fad_last_error(void) { return g_err.c_str(); }

int fad_create(int device, int max_examples, fad_handle** out) {
    if (!out) return fail("null out pointer");
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0)
        return fail("no CUDA device: fadtk_b200 has no CPU fallback");
    if (device < 0 || device >= count) return fail("bad device index");
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9) return fail("fadtk_b200 kernels are built for sm_90a (Hopper H100) only");
    std::unique_ptr<fad_handle> h(new fad_handle());
    h->device = device;
    h->num_sms = prop.multiProcessorCount;
    h->max_examples = max_examples > 0 ? max_examples : 2048;

    std::vector<double> tw, hann, melw; std::vector<int> ms, mc;
    build_frontend_tables(tw, hann, melw, ms, mc);
    if (upload(h->mem, &h->d_twiddle, tw.data(), tw.size() * 8) || upload(h->mem, &h->d_hann, hann.data(), hann.size() * 8) ||
        upload(h->mem, &h->d_melw, melw.data(), melw.size() * 8) || upload(h->mem, &h->d_mel_start, ms.data(), ms.size() * 4) ||
        upload(h->mem, &h->d_mel_count, mc.data(), mc.size() * 4)) return 1;
    // one-time kernel setup, for the handle's device: the dynamic shared memory of every kernel that launches with more
    // than the default 48 KiB, and the GEMM's co-resident CTA pairs
    const auto smem = [](const void* kernel, size_t bytes) {
        return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    };
    CK(smem((const void*)fad::logmel_kernel<double>, fad::logmel_smem_bytes<double>()));
    CK(smem((const void*)fad::logmel_kernel<float>, fad::logmel_smem_bytes<float>()));
    CK(smem((const void*)fad::clap_logmel_kernel, fad::clap_logmel_smem_bytes()));
    CK(smem((const void*)fad::attention_wgmma_kernel, fad::kAtSmem));
    CK(smem((const void*)fad::clap_window_attention_kernel<24>, fad::att_smem_bytes(24, fad::kAttWarps, fad::kAttStages)));
    CK(smem((const void*)fad::clap_window_attention_kernel<32>, fad::att_smem_bytes(32, fad::kAttWarps, fad::kAttStages)));
    CK(smem((const void*)fad::kad_tile_kernel<0>, fad::kKadSmemBytes));
    CK(smem((const void*)fad::kad_tile_kernel<1>, fad::kKadSmemBytes));
    CK(smem((const void*)fad::kad_tile_kernel<2>, fad::kKadSmemBytes));
    CK(smem((const void*)fad::kad_perm_tile_kernel<false>, fad::kPermSmemBytes));
    CK(smem((const void*)fad::kad_perm_tile_kernel<true>, fad::kPermSmemBytes));
    CK(smem((const void*)fad::prdc_tile_kernel<0>, fad::kPairSmemBytes));
    CK(smem((const void*)fad::prdc_tile_kernel<1>, fad::kPairSmemBytes));
    CK(smem((const void*)fad::prdc_tile_kernel<2>, fad::kPairSmemBytes));
    CK(smem((const void*)fad::prdc_tile_kernel<3>, fad::kPrdcSongSmemBytes));
    CK(smem((const void*)fad::prdc_tile_kernel<4>, fad::kPairSmemBytes));
    CK(smem((const void*)fad::prdc_tile_kernel<5>, fad::kPrdcNearestSmemBytes));
    CK(smem((const void*)fad::prdc_tile_kernel<6>, fad::kPairSmemBytes));
    if (setup_gemm<0>(h.get()) || setup_gemm<1>(h.get())) return 1;
    *out = h.release();
    return 0;
}

int fad_destroy(fad_handle* h) {
    if (!h) return 0;
    cudaSetDevice(h->device);
    fad_comm_destroy(h);
    delete h;
    return 0;
}

long long fad_launch_count(fad_handle* h) { return h ? h->launches : 0; }

// ------------------------------------------------------------------------------ VGGish
int fad_vggish_load(fad_handle* h, const fad_vggish_weights* w) {
    if (!h || !w) return fail("null argument");
    // conv1's weight and bias, then the weights and the biases of the kVgg layers
    const void* src[18] = {w->conv1_w_host, w->conv1_b_host,
                           w->conv_w_host[0], w->conv_w_host[1], w->conv_w_host[2], w->conv_w_host[3], w->conv_w_host[4],
                           w->fc_w_host[0], w->fc_w_host[1], w->fc_w_host[2],
                           w->conv_b_host[0], w->conv_b_host[1], w->conv_b_host[2], w->conv_b_host[3], w->conv_b_host[4],
                           w->fc_b_host[0], w->fc_b_host[1], w->fc_b_host[2]};
    if (check_tensors("fad_vggish_load", src, 18)) return 1;
    const void* const* wsrc = src + 2;
    const void* const* bsrc = src + 10;
    CK(cudaSetDevice(h->device));
    h->vgg.reset();
    auto vs = std::make_unique<VggState>();
    auto& m = vs->mem;
    if (upload(m, &vs->conv1_w, src[0], 64 * 9 * 4) || upload(m, &vs->conv1_b, src[1], 64 * 4)) return 1;
    for (int i = 0; i < 8; ++i) {
        const VggLayer& L = kVgg[i];
        const size_t mul = ((w->split_mask >> i) & 1) ? 2 : 1;      // sizes depend on split_mask
        if (upload(m, &vs->w[i], wsrc[i], mul * L.Cout * L.taps * L.Cin * 2) || upload(m, &vs->b[i], bsrc[i], (size_t)L.Cout * 4))
            return 1;
    }
    for (int i = 0; i < 8; ++i)
        if (((w->split_mask >> i) & 1) &&
            note_split_weights(h, vs->w[i], kVgg[i].Cout / 128, (long long)kVgg[i].taps * kVgg[i].Cin, 0)) return 1;
    const size_t B = (size_t)h->max_examples;
    if (alloc(m, &vs->logmel, B * 96 * 64 * 4)) return 1;
    for (int i = 0; i < 8; ++i)
        if (alloc(m, &vs->act[i], B * kActElems[i] * 2)) return 1;
    // descriptors of the fixed pipeline (batch dimension = max_examples; tiles past the live
    // batch are never scheduled and rows past it are masked in the epilogue)
    for (int i = 0; i < 8; ++i) {
        const VggLayer& L = kVgg[i];
        if (make_geom(vs->geom[i], L.H, L.W, L.Cin, L.Cout, L.taps, L.relu, L.pool, (w->split_mask >> i) & 1)) return 1;
        if (encode_layer_maps(vs->geom[i], vs->act[i], (long long)B, vs->w[i], &vs->map_x[i], &vs->map_w[i])) return 1;
    }
    h->vgg = std::move(vs);
    return 0;
}

long long fad_vggish_num_examples(long long n_samples) {
    if (n_samples < fad::kWin) return 0;
    const long long t = 1 + (n_samples - fad::kWin) / fad::kHop;
    if (t < fad::kExFrames) return 0;
    return 1 + (t - fad::kExFrames) / fad::kExFrames;
}

long long fad_vggish_plan(const long long* clip_offsets_host, long long n_clips,
                          long long* ex_start_host, long long capacity, long long* rows_per_clip_host) {
    long long n = 0;
    for (long long c = 0; c < n_clips; ++c) {
        const long long len = clip_offsets_host[c + 1] - clip_offsets_host[c];
        const long long k = fad_vggish_num_examples(len);
        if (rows_per_clip_host) rows_per_clip_host[c] = k;
        for (long long e = 0; e < k; ++e, ++n)
            if (ex_start_host && n < capacity)
                ex_start_host[n] = clip_offsets_host[c] + e * (long long)(fad::kExFrames * fad::kHop);
    }
    return n;
}

static int launch_logmel(fad_handle* h, const int16_t* pcm, const long long* ex_start, long long n,
                         float* out, int use_double, cudaStream_t st) {
    fad::FrontendTables tab{h->d_twiddle, h->d_hann, h->d_melw, h->d_mel_start, h->d_mel_count};
    const long long frames = n * fad::kExFrames;
    long long blocks = (frames + fad::kFeWarps - 1) / fad::kFeWarps;
    const long long cap = (long long)h->num_sms * 8;
    if (blocks > cap) blocks = cap;
    if (use_double)
        return launch(h, fad::logmel_kernel<double>, (int)blocks, fad::kFeWarps * 32, fad::logmel_smem_bytes<double>(), st,
                      pcm, ex_start, (int)n, tab, out);
    return launch(h, fad::logmel_kernel<float>, (int)blocks, fad::kFeWarps * 32, fad::logmel_smem_bytes<float>(), st,
                  pcm, ex_start, (int)n, tab, out);
}

int fad_vggish_logmel(fad_handle* h, const int16_t* pcm, const long long* ex_start,
                      long long n_examples, float* logmel_out, int use_double, void* stream) {
    if (!h) return fail("null handle");
    CK(cudaSetDevice(h->device));
    return launch_logmel(h, pcm, ex_start, n_examples, logmel_out, use_double, (cudaStream_t)stream);
}

int fad_vggish_forward(fad_handle* h, const int16_t* pcm, const long long* ex_start,
                       long long n_examples, void* emb_out_f16, void* stream) {
    if (!h) return fail("null handle");
    if (!h->vgg) return fail("fad_vggish_load has not been called");
    CK(cudaSetDevice(h->device));
    const VggState& vs = *h->vgg;
    cudaStream_t st = (cudaStream_t)stream;
    static const int fe_double = []() { const char* e = getenv("FADTK_FRONTEND_FP64"); return (e && e[0] == '1') ? 1 : 0; }();
    for (long long base = 0; base < n_examples; base += h->max_examples) {
        const int nb = (int)((n_examples - base) < h->max_examples ? (n_examples - base) : h->max_examples);
        size_t ev = prof_begin(h, st);
        if (launch_logmel(h, pcm, ex_start + base, nb, vs.logmel, fe_double, st)) return 1;
        prof_end(h, FAD_PROF_LOGMEL, ev, st);
        ev = prof_begin(h, st);
        if (launch(h, fad::conv1_kernel, dim3(6, nb), 256, 0, st, vs.logmel, vs.conv1_w, vs.conv1_b, vs.act[0])) return 1;
        prof_end(h, FAD_PROF_CONV1, ev, st);
        for (int i = 0; i < 8; ++i) {
            void* out = (i == 7) ? (void*)((__half*)emb_out_f16 + (size_t)base * 128) : (void*)vs.act[i + 1];
            ev = prof_begin(h, st);
            if (run_layer(h, vs.geom[i], vs.map_x[i], vs.map_w[i], vs.w[i], nb, vs.b[i], out, nullptr, st)) return 1;
            prof_end(h, FAD_PROF_LAYER0 + i, ev, st);
        }
    }
    return 0;
}

// Stage entry (parity test): conv1 (3x3, 1 -> 64, pad 1) + bias + ReLU + 2x2 max-pool on fp32 log-mel examples.
int fad_vggish_conv1(fad_handle* h, const float* logmel, long long n_examples, void* out_f16, void* stream) {
    if (!h) return fail("null handle");
    if (!h->vgg) return fail("fad_vggish_load has not been called");
    if (n_examples <= 0) return 0;
    CK(cudaSetDevice(h->device));
    return launch(h, fad::conv1_kernel, dim3(6, (unsigned)n_examples), 256, 0, (cudaStream_t)stream,
                  logmel, h->vgg->conv1_w, h->vgg->conv1_b, reinterpret_cast<__half*>(out_f16));
}

int fad_umma_layer(fad_handle* h, const void* x_f16, int NB, int H, int W, int Cin,
                   const void* w_f16, const float* bias, int Cout, int taps, int relu, int pool,
                   int split_w, void* out_f16, float* out_f32_or_null, void* stream) {
    if (!h) return fail("null handle");
    if (split_w != 0 && split_w != 1) return fail("fad_umma_layer: split_w must be 0 (fp16 weights) or 1 (fp16 hi/lo pair)");
    CK(cudaSetDevice(h->device));
    LayerGeom g;
    if (make_geom(g, H, W, Cin, Cout, taps, relu, pool, split_w)) return 1;
    if (pool && out_f32_or_null) return fail("fp32 copy is only available for un-pooled layers");
    if (g.split_w == 1 && note_split_weights(h, w_f16, Cout / 128, (long long)taps * Cin, (cudaStream_t)stream)) return 1;
    CUtensorMap mx, mw;
    if (encode_layer_maps(g, x_f16, NB, w_f16, &mx, &mw)) return 1;
    return run_layer(h, g, mx, mw, w_f16, NB, bias, out_f16, out_f32_or_null, (cudaStream_t)stream);
}

// -------------------------------------------------------------------------- statistics
size_t fad_stats_acc_len(int d) { return 1 + 2 * (size_t)d + (size_t)d * d; }

int fad_stats_accumulate(fad_handle* h, const void* emb_f16, long long n_rows, int d,
                         const void* shift_f16, double* acc, int tensor_core, void* stream) {
    if (!h) return fail("null handle");
    // 0: exact fp64 Gram on the FP64 tensor pipe (DMMA), the product path; 2: fp64 CUDA-core kernel (cross-check)
    if (tensor_core != 0 && tensor_core != 2) return fail("fad_stats_accumulate: tensor_core must be 0 (DMMA) or 2 (CUDA-core fp64)");
    if (n_rows <= 0) return 0;
    CK(cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    const __half* E = reinterpret_cast<const __half*>(emb_f16);
    const __half* shift = reinterpret_cast<const __half*>(shift_f16);
    if (tensor_core == 0) return launch_stats_dmma(h, E, n_rows, d, shift, acc, st);
    if (d % 64 != 0) return fail("d must be a multiple of 64");
    dim3 grid((unsigned)((n_rows + fad::kSimtRows - 1) / fad::kSimtRows), d / 64, d / 64);
    return launch(h, fad::stats_simt_kernel, grid, 256, 0, st, E, n_rows, d, shift, acc);
}

// ---- the reference's per-file statistics semantics for equal-length files, on the device (fadtk/utils.py:13-46) ----
int fad_file_means(fad_handle* h, const void* emb_f16, long long n_files, int rows_per_file, int d,
                   double* m64_out, double* m16_out, void* stream) {
    if (!h) return fail("null handle");
    if (n_files <= 0) return 0;
    if (rows_per_file <= 0 || d <= 0) return fail("bad shape");
    CK(cudaSetDevice(h->device));
    long long blocks = (n_files * d + 255) / 256;
    if (blocks > (long long)h->num_sms * 16) blocks = (long long)h->num_sms * 16;
    return launch(h, fad::file_means_kernel, (unsigned)blocks, 256, 0, (cudaStream_t)stream,
                  reinterpret_cast<const __half*>(emb_f16), n_files, rows_per_file, d, m64_out, m16_out);
}

// exact Gram statistics of fp64 rows (no shift): acc[0] += n, acc[1..d] += sum x, outer += sum x x^T (DMMA, fixed order)
int fad_stats_accumulate_f64(fad_handle* h, const double* rows, long long n_rows, int d, double* acc, void* stream) {
    if (!h) return fail("null handle");
    if (n_rows <= 0) return 0;
    CK(cudaSetDevice(h->device));
    return launch_stats_dmma(h, rows, n_rows, d, nullptr, acc, (cudaStream_t)stream);
}

int fad_stats_finalize_mirrored(fad_handle* h, const double* acc, const double* acc_means64, const double* acc_means16,
                                const void* shift_f16, int rows_per_file, int d, double* mu_out, double* cov_out, void* stream) {
    if (!h) return fail("null handle");
    CK(cudaSetDevice(h->device));
    static const int keep = [] { const char* e = getenv("FADTK_SINGLE_FRAME_FILES"); return (e && std::string(e) == "keep") ? 1 : 0; }();
    const size_t total = (size_t)d * d;
    unsigned blocks = (unsigned)((total + 255) / 256);
    if (blocks > (unsigned)h->num_sms * 8) blocks = h->num_sms * 8;
    return launch(h, fad::stats_finalize_mirrored_kernel, blocks, 256, 0, (cudaStream_t)stream,
                  acc, acc_means64, acc_means16, reinterpret_cast<const __half*>(shift_f16), rows_per_file, d, keep, mu_out, cov_out);
}

int fad_stats_accumulate_gather(fad_handle* h, const void* emb_f16, long long n_src_rows,
                                const long long* idx, long long n_idx, int d,
                                const void* shift_f16, double* acc, void* stream) {
    if (!h) return fail("null handle");
    (void)n_src_rows;
    if (n_idx <= 0) return 0;
    if (d % 8 != 0) return fail("d must be a multiple of 8");
    CK(cudaSetDevice(h->device));
    if (h->gather_buf.grow((size_t)n_idx * d * 2)) return 1;
    __half* rows = h->gather_buf.get<__half>();
    const long long vecs = n_idx * (d / 8);
    long long blocks = (vecs + 255) / 256;
    if (blocks > (long long)h->num_sms * 16) blocks = (long long)h->num_sms * 16;
    if (launch(h, fad::gather_rows_kernel, (unsigned)blocks, 256, 0, (cudaStream_t)stream,
               reinterpret_cast<const __half*>(emb_f16), idx, n_idx, d, rows)) return 1;
    return launch_stats_dmma(h, rows, n_idx, d, reinterpret_cast<const __half*>(shift_f16), acc, (cudaStream_t)stream);
}

int fad_stats_finalize(fad_handle* h, const double* acc, const void* shift_f16, int d,
                       double* mu_out, double* cov_out, void* stream) {
    if (!h) return fail("null handle");
    CK(cudaSetDevice(h->device));
    const size_t total = (size_t)d * d;
    unsigned blocks = (unsigned)((total + 255) / 256);
    if (blocks > (unsigned)h->num_sms * 8) blocks = h->num_sms * 8;
    return launch(h, fad::stats_finalize_kernel, blocks, 256, 0, (cudaStream_t)stream,
                  acc, reinterpret_cast<const __half*>(shift_f16), d, mu_out, cov_out);
}

// Stage entry (parity test): encoder self-attention of n_clips sequences of S positions, heads of 64 dims.
// qkv fp16 [n_clips * S][3 d] (q | k | v), out fp16 [n_clips * S][d]; legacy != 0 runs the mma.sync kernel instead.
extern "C" int fad_attention(fad_handle* h, const void* qkv_f16, long long n_clips, int S, int d, void* out_f16, int legacy, void* stream) {
    if (!h || !qkv_f16 || !out_f16) return fail("null argument");
    if (d % 64 != 0 || S <= 0 || n_clips <= 0) return fail("bad shape");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (!legacy) return launch_attention_wgmma(h, reinterpret_cast<const __half*>(qkv_f16), n_clips, S, d, d / 64, reinterpret_cast<__half*>(out_f16), st);
    return launch(h, fad::whisper_flash_attention_kernel, dim3((S + 63) / 64, d / 64, (unsigned)n_clips), 128, 0, st,
                  reinterpret_cast<const __half*>(qkv_f16), S, d, reinterpret_cast<__half*>(out_f16), nullptr, nullptr);
}


// ------------------------------------------------------------------- cross-GPU statistics merge
// The one exchange step of the path (SURVEY.md section 8 (e)): all-reduce(sum) of the packed fp64 accumulator over
// NVLink.  NCCL is resolved at run time with dlopen (the process usually has torch's libnccl.so.2 mapped already;
// $FADTK_NCCL_LIB overrides) so the library keeps loading on hosts without NCCL and links nothing but the C++ runtime.
#include <dlfcn.h>
namespace {
struct NcclId { char bytes[128]; };
struct NcclApi {
    int (*GetUniqueId)(NcclId*) = nullptr;
    int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*CommCount)(void*, int*) = nullptr;
    int (*CommUserRank)(void*, int*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
    std::string why;
};
NcclApi& nccl_api() {
    static NcclApi api = [] {
        NcclApi a;
        const char* env = getenv("FADTK_NCCL_LIB");
        const char* names[] = {env, "libnccl.so.2", "libnccl.so"};
        void* lib = nullptr;
        for (const char* n : names) {
            if (!n || !*n) continue;
            lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (lib) break;
        }
        if (!lib) { a.why = "libnccl.so.2 not found (set FADTK_NCCL_LIB)"; return a; }
        a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(lib, "ncclGetUniqueId"));
        a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(lib, "ncclCommInitRank"));
        a.AllReduce = reinterpret_cast<decltype(a.AllReduce)>(dlsym(lib, "ncclAllReduce"));
        a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
        a.CommCount = reinterpret_cast<decltype(a.CommCount)>(dlsym(lib, "ncclCommCount"));
        a.CommUserRank = reinterpret_cast<decltype(a.CommUserRank)>(dlsym(lib, "ncclCommUserRank"));
        a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
        a.ok = a.GetUniqueId && a.CommInitRank && a.AllReduce && a.CommDestroy && a.CommCount && a.CommUserRank &&
               a.GetErrorString;
        if (!a.ok) a.why = "NCCL library lacks an expected symbol";
        return a;
    }();
    return api;
}
int nccl_fail(const char* what, int rc) {
    return fail(std::string(what) + ": " + (nccl_api().GetErrorString ? nccl_api().GetErrorString(rc) : "NCCL error"));
}
}  // namespace

extern "C" {
int fad_comm_unique_id(void* id_out_host) {
    if (!id_out_host) return fail("null argument");
    NcclApi& n = nccl_api();
    if (!n.ok) return fail(n.why);
    NcclId id;
    const int rc = n.GetUniqueId(&id);
    if (rc != 0) return nccl_fail("ncclGetUniqueId", rc);
    memcpy(id_out_host, id.bytes, sizeof id.bytes);
    return 0;
}

int fad_comm_init(fad_handle* h, const void* id_host, int rank, int world) {
    if (!h || !id_host) return fail("null argument");
    if (world < 1 || rank < 0 || rank >= world) return fail("bad rank / world size");
    NcclApi& n = nccl_api();
    if (!n.ok) return fail(n.why);
    CK(cudaSetDevice(h->device));
    if (h->nccl_comm) { n.CommDestroy(h->nccl_comm); h->nccl_comm = nullptr; }
    NcclId id;
    memcpy(id.bytes, id_host, sizeof id.bytes);
    const int rc = n.CommInitRank(&h->nccl_comm, world, id, rank);
    if (rc != 0) { h->nccl_comm = nullptr; return nccl_fail("ncclCommInitRank", rc); }
    return 0;
}

int fad_comm_destroy(fad_handle* h) {
    if (h && h->nccl_comm) { nccl_api().CommDestroy(h->nccl_comm); h->nccl_comm = nullptr; }
    return 0;
}

int fad_allreduce_sum_f64(fad_handle* h, void* nccl_comm_or_null, double* buf, long long n_values, void* stream) {
    if (!h || !buf) return fail("null argument");
    void* comm = nccl_comm_or_null ? nccl_comm_or_null : h->nccl_comm;
    if (!comm) return fail("no communicator: call fad_comm_init or pass an ncclComm_t");
    NcclApi& n = nccl_api();
    if (!n.ok) return fail(n.why);
    CK(cudaSetDevice(h->device));
    const int rc = n.AllReduce(buf, buf, (size_t)n_values, /*ncclFloat64*/ 8, /*ncclSum*/ 0, comm, (cudaStream_t)stream);
    if (rc != 0) return nccl_fail("ncclAllReduce", rc);
    return 0;
}

int fad_stats_allreduce(fad_handle* h, void* nccl_comm_or_null, double* acc, int d, void* stream) {
    if (d <= 0) return fail("bad dimension");
    return fad_allreduce_sum_f64(h, nccl_comm_or_null, acc, (long long)fad_stats_acc_len(d), stream);
}
}  // extern "C"

// ----------------------------------------------------------------------------- Frechet
namespace {
// carve-outs of h->fr_buf for a group of G items of d x d problems
struct FrechetWorkspace {
    double *cov, *P, *M, *Y, *Z, *W, *Yn, *Zn;  // [G][d][d] each
    double* mu;                                // [G][d]
    double *scalC, *scalM;                     // [G][2]: {|A|_F, tr A} of C2_z and of M_z
    float* flags;                              // [G][3]: rotating max |W - I| slots of the chain
    int* ok;                                   // [G]: item has >= 2 rows
    double* sqrt1;                             // [d][d]: fad_frechet's C1^(1/2)
    double* scal1;                             // [2]: fad_frechet's {|C1|_F, tr C1}
    double* resid;                             // [1]: |Y Y - Mn|_F^2 of one item
    double* sink;                              // [1]: keeps dmma_peak_kernel's result alive
};

int frechet_workspace(fad_handle* h, long long G, int d, FrechetWorkspace& w) {
    const size_t mat = G * (size_t)d * d;
    if (carve(h->fr_buf, slot(w.cov, mat), slot(w.P, mat), slot(w.M, mat), slot(w.Y, mat), slot(w.Z, mat), slot(w.W, mat),
              slot(w.Yn, mat), slot(w.Zn, mat), slot(w.mu, G * d), slot(w.scalC, G * 2), slot(w.scalM, G * 2),
              slot(w.flags, G * 3), slot(w.ok, G), slot(w.sqrt1, (size_t)d * d), slot(w.scal1, 4))) return 1;
    w.resid = w.scal1 + 2;
    w.sink = w.scal1 + 3;
    return 0;
}

// grid of the elementwise d x d kernels: one item spreads over the whole GPU
unsigned elem_blocks(const fad_handle* h, int d) {
    const size_t b = ((size_t)d * d + 255) / 256;
    return (unsigned)std::min(b, (size_t)h->num_sms * 8);
}

int launch_dgemm(fad_handle* h, const fad::DgemmStrided& p, int families, int d, cudaStream_t st) {
    dim3 grid((d + fad::kDgTileN - 1) / fad::kDgTileN, (d + fad::kDgTileM - 1) / fad::kDgTileM, (unsigned)(p.items * families));
    return launch(h, fad::dgemm_strided_kernel, grid, 256, 0, st, p, d);
}

// Coupled Newton-Schulz on the g matrices A_z: on return w.Y_z ~ sqrt(sym(A_z)/|A_z|_F + delta I), w.Z_z its
// inverse, scal[z] = {|A_z|_F, tr A_z}.
int newton_schulz(fad_handle* h, const FrechetWorkspace& w, const double* A, double* scal, int g, int d, int iters,
                  cudaStream_t st) {
    if (launch(h, fad::norm_trace_kernel, g, 1024, 0, st, A, d, scal) ||
        launch(h, fad::ns_init_kernel, dim3(elem_blocks(h, d), g), 256, 0, st, A, d, scal, w.Y, w.Z, w.flags)) return 1;
    // (Y, Z) <-> (Yn, Zn) ping-pong on a fixed host schedule; an even iteration count lands the
    // last scheduled update in (Y, Z).  If an item stops early (dev < tol) the two pairs differ by
    // one factor W with |W - I| < tol, i.e. by < 1e-12 relative - either is the converged iterate.
    if (iters & 1) ++iters;
    const long long T = (long long)d * d;
    double *Yc = w.Y, *Zc = w.Z, *Yx = w.Yn, *Zx = w.Zn;
    for (int it = 0; it < iters; ++it) {
        fad::DgemmStrided wp = {};
        wp.items = g; wp.flags = w.flags; wp.tol = 1e-12f;
        wp.in_slot = (it + 2) % 3; wp.out_slot = it % 3; wp.clear_slot = -1;     // slots: iteration it-1, it, it+1
        wp.f[0] = {Zc, Yc, w.W, T, T, T, -0.5, 1.5};                             // W = 1.5 I - 0.5 Z Y
        if (launch_dgemm(h, wp, 1, d, st)) return 1;
        fad::DgemmStrided yz = wp;
        yz.out_slot = -1; yz.clear_slot = (it + 1) % 3;
        yz.f[0] = {Yc, w.W, Yx, T, T, T, 1.0, 0.0};                              // Y <- Y W
        yz.f[1] = {w.W, Zc, Zx, T, T, T, 1.0, 0.0};                              // Z <- W Z
        if (launch_dgemm(h, yz, 2, d, st)) return 1;
        std::swap(Yc, Yx);
        std::swap(Zc, Zx);
    }
    return 0;
}

// FAD of g eval sets (mu2_z, C2_z) against the baseline (mu1, S = C1^(1/2), scal1 = {|C1|_F, tr C1}) into out[z][8]:
// P = S C2_z, M_z = P S, the chain on M_z, the assembly.  out[z][3] reports `iters` as given.  With_resid (one item)
// puts the relative residual of the square root in out[0][2]: P = Y Y, then resid_kernel.
int frechet_items(fad_handle* h, const FrechetWorkspace& w, const double* mu1, const double* sqrt1, const double* scal1,
                  const double* mu2, const double* cov2, int g, int d, int iters, const int* ok,
                  const long long* offsets, bool with_resid, double* out, cudaStream_t st) {
    const long long T = (long long)d * d;
    if (launch(h, fad::norm_trace_kernel, g, 1024, 0, st, cov2, d, w.scalC)) return 1;
    fad::DgemmStrided p = {};
    p.items = g; p.in_slot = p.out_slot = p.clear_slot = -1;
    p.f[0] = {sqrt1, cov2, w.P, 0, T, T, 1.0, 0.0};                                 // P = S C2_z
    if (launch_dgemm(h, p, 1, d, st)) return 1;
    p.f[0] = {w.P, sqrt1, w.M, T, 0, T, 1.0, 0.0};                                  // M_z = P S
    if (launch_dgemm(h, p, 1, d, st)) return 1;
    if (newton_schulz(h, w, w.M, w.scalM, g, d, iters, st)) return 1;
    if (with_resid) {
        CK(cudaMemsetAsync(w.resid, 0, sizeof(double), st));
        p.f[0] = {w.Y, w.Y, w.P, T, T, T, 1.0, 0.0};                                // P = Y Y
        if (launch_dgemm(h, p, 1, d, st)) return 1;
        if (launch(h, fad::resid_kernel, elem_blocks(h, d), 256, 0, st, w.P, w.M, d, w.scalM, w.resid)) return 1;
    }
    return launch(h, fad::frechet_assemble_kernel, g, 256, 0, st, mu1, mu2, d, scal1, w.scalC, w.scalM, w.Y, w.Z,
                  with_resid ? w.resid : nullptr, ok, offsets, iters, out);
}
}  // namespace

// S = C^(1/2) and tr C of a baseline covariance, computed once and reused for every eval set
// (FAD-inf steps, per-song scores).  sqrt_out: d*d doubles, scal_out: 2 doubles (|C|_F, tr C), device.
int fad_sqrt_psd(fad_handle* h, const double* cov, int d, int iters, double* sqrt_out, double* scal_out,
                 void* stream) {
    if (!h) return fail("null handle");
    if (d <= 0) return fail("bad dimension");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (iters <= 0) iters = 60;
    FrechetWorkspace w;
    if (frechet_workspace(h, 1, d, w)) return 1;
    const size_t ev = prof_begin(h, st);
    if (newton_schulz(h, w, cov, w.scalC, 1, d, iters, st)) return 1;
    if (launch(h, fad::ns_unscale_kernel, elem_blocks(h, d), 256, 0, st, w.Y, d, w.scalC, sqrt_out)) return 1;
    CK(cudaMemcpyAsync(scal_out, w.scalC, 2 * sizeof(double), cudaMemcpyDeviceToDevice, st));
    prof_end(h, FAD_PROF_FRECHET, ev, st);
    return 0;
}

// FAD against a baseline given by (mu1, S1 = C1^(1/2), scal1 = {|C1|_F, tr C1}).
int fad_frechet_presqrt(fad_handle* h, const double* mu1, const double* sqrt1, const double* scal1,
                        const double* mu2, const double* cov2, int d, int iters, double* out, void* stream) {
    if (!h) return fail("null handle");
    if (d <= 0) return fail("bad dimension");
    CK(cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (iters <= 0) iters = 60;
    FrechetWorkspace w;
    if (frechet_workspace(h, 1, d, w)) return 1;
    const size_t ev = prof_begin(h, st);
    if (frechet_items(h, w, mu1, sqrt1, scal1, mu2, cov2, 1, d, iters, nullptr, nullptr, true, out, st)) return 1;
    prof_end(h, FAD_PROF_FRECHET, ev, st);
    return 0;
}

int fad_frechet(fad_handle* h, const double* mu1, const double* cov1, const double* mu2,
                const double* cov2, int d, int iters, double* out, void* stream) {
    if (!h) return fail("null handle");
    if (d <= 0) return fail("bad dimension");
    CK(cudaSetDevice(h->device));
    FrechetWorkspace w;                   // the same carve-out as the two calls below: S and scal1 stay put
    if (frechet_workspace(h, 1, d, w)) return 1;
    if (fad_sqrt_psd(h, cov1, d, iters, w.sqrt1, w.scal1, stream)) return 1;
    return fad_frechet_presqrt(h, mu1, w.sqrt1, w.scal1, mu2, cov2, d, iters, out, stream);
}

// Ragged-batched FAD of n_items eval sets against one cached baseline: per-song statistics (stats.cuh), then the
// chain over groups of up to G items.
int fad_frechet_batched(fad_handle* h, const double* mu1, const double* sqrt1, const double* scal1,
                        const void* emb_f16, const long long* offsets, long long n_items, int d, int iters,
                        double* out, void* stream) {
    if (!h) return fail("null handle");
    if (d <= 0 || n_items < 0) return fail("bad dimension");
    if (n_items == 0) return 0;
    CK(cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (iters <= 0) iters = 60;
    if (iters & 1) ++iters;                                                // out[z][3]: the even count the chain runs
    long long G = (long long)((size_t(1) << 31) / (64 * (size_t)d * d));  // 8 matrices of d*d doubles per item in 2 GiB
    if (G < 1) G = 1;
    if (G > 32767) G = 32767;                                              // two families share gridDim.z
    if (G > n_items) G = n_items;
    FrechetWorkspace w;
    if (frechet_workspace(h, G, d, w)) return 1;
    const __half* emb = reinterpret_cast<const __half*>(emb_f16);
    const size_t ev = prof_begin(h, st);
    for (long long g0 = 0; g0 < n_items; g0 += G) {
        const int g = (int)((n_items - g0) < G ? (n_items - g0) : G);
        const int nt = d / 64, dt = (d + 31) / 32;
        if (d % 64 == 0 ?                                    // fp64 tensor pipe (DMMA), upper tile triangle per item
                launch(h, fad::song_stats_dmma_kernel, dim3(nt * (nt + 1) / 2, g), 256, 0, st, emb, offsets + g0, d, w.mu, w.cov, w.ok) :
                launch(h, fad::song_stats_kernel, dim3(dt, dt, g), 256, 0, st, emb, offsets + g0, d, w.mu, w.cov, w.ok))
            return 1;
        if (frechet_items(h, w, mu1, sqrt1, scal1, w.mu, w.cov, g, d, iters, w.ok, offsets + g0, false, out + g0 * 8, st))
            return 1;
    }
    prof_end(h, FAD_PROF_FRECHET, ev, st);
    return 0;
}

// ------------------------------------------------------------------- fp64 tensor-pipe peak
// Roofline denominator of the DMMA kernels (exact Gram, Newton-Schulz): MEASURED_PEAKS.json only
// carries the bf16 GEMM and HBM copy rates, so the fp64 tensor-pipe rate is measured here - every warp
// of a full grid issues independent m8n8k4 DMMAs from registers, nothing else.
namespace {
__global__ void __launch_bounds__(256) dmma_peak_kernel(int iters, double* sink) {
    double c[8][2];
#pragma unroll
    for (int i = 0; i < 8; ++i) { c[i][0] = threadIdx.x; c[i][1] = -1.0 * threadIdx.x; }
    const double a = 1.0 + 1e-9 * threadIdx.x, b = 1.0 - 1e-9 * threadIdx.x;
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) sm90::dmma_884(c[i][0], c[i][1], a, b);
    }
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1];
    if (s == 12345.678) sink[0] = s;                       // keeps the chain alive, never true
}
}  // namespace

extern "C" int fad_bench_dmma_peak(fad_handle* h, int iters, double* tflops_out_host) {
    if (!h || !tflops_out_host) return fail("null argument");
    CK(cudaSetDevice(h->device));
    if (iters <= 0) iters = 20000;
    FrechetWorkspace w;
    if (frechet_workspace(h, 1, 1, w)) return 1;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const int blocks = h->num_sms * 4;
    if (launch(h, dmma_peak_kernel, blocks, 256, 0, nullptr, iters / 10, w.sink)) return 1;     // warm-up
    CK(cudaEventRecord(e0));
    if (launch(h, dmma_peak_kernel, blocks, 256, 0, nullptr, iters, w.sink)) return 1;
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    const double flop = (double)blocks * 8 /*warps*/ * (double)iters * 8 /*DMMAs*/ * 512.0;
    *tflops_out_host = flop / (ms * 1e-3) / 1e12;
    return 0;
}
}  // extern "C"

#include "pairwise_host.inc"
#include "fad_test_host.inc"
#include "bootstrap_host.inc"

#include "resample_host.inc"
#include "clap_host.inc"

extern "C" int fad_linear(fad_handle* h, const void* a_f16, long long rows, int k_cols, long long lda, const void* w_f16,
                          int split_w, const float* bias, int n_cols, int act, void* out_f16, float* out_f32,
                          float* resid, int resid_C, int resid_res, int resid_shift, void* stream) {
    if (!h) return fail("null handle");
    CK(cudaSetDevice(h->device));
    const __half* A = reinterpret_cast<const __half*>(a_f16);
    const __half* W = reinterpret_cast<const __half*>(w_f16);
    __half* out16 = reinterpret_cast<__half*>(out_f16);
    if (clap_gemm_check(A, rows, k_cols, W, bias, n_cols, act, out16, out_f32, resid, resid_C, resid_res, resid_shift, lda, split_w))
        return 1;
    // the caller's weights: whether their lo parts are zero is decided on every call, never taken from a cache
    if (split_w == 1 && note_split_weights(h, W, pad_to(n_cols, 128) / 128, pad_to(k_cols, 64), (cudaStream_t)stream)) return 1;
    return clap_gemm(h, A, rows, k_cols, W, bias, n_cols, act, out16, out_f32, (cudaStream_t)stream,
                     resid, resid_C, resid_res, resid_shift, lda, split_w);
}

#include "whisper_host.inc"
#include "encodec_host.inc"
#include "wav2vec_host.inc"

fad_handle::~fad_handle() = default;
