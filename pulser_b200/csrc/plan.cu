// Host side of the C ABI (include/pulser_b200.h): plan, interpolation tables,
// Magnus/Chebyshev schedule, kernel launches.
//
// Algorithm (DESIGN.md section 3): the sampling grid is cut into Magnus steps
// [a, b]; on each step the exact moments B0 = int H dt and
// B1 = (1/h) int (t - t_mid) H dt of the *interpolated* coefficient functions
// define the 4th-order commutator-free propagator
//     psi <- exp(-i(B0/2 + 2 B1)) exp(-i(B0/2 - 2 B1)) psi ,
// and each exponential is a Chebyshev expansion evaluated with the Clenshaw
// recurrence, one fused H-apply kernel per term.
#include <cuda_runtime.h>

#include <algorithm>
#include <deque>
#include <map>
#include <memory>
#include <mutex>
#include <unordered_map>
#include <cmath>
#include <complex>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/pulser_b200.h"
#include "kernels.cuh"
#include "spline.hpp"
#include <cub/device/device_scan.cuh>
#include <nvtx3/nvToolsExt.h>
#include <random>

namespace pb200 {

static thread_local std::string g_last_error;

struct Error : std::runtime_error {
    int code;
    Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

[[noreturn]] static void fail(int code, const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    throw Error(code, buf);
}

#define CUDA_CHECK(expr)                                                                        \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess)                                                                 \
            fail(PB200_ERR_CUDA, "CUDA error %s at %s:%d: %s", #expr, __FILE__, __LINE__,       \
                 cudaGetErrorString(e__));                                                      \
    } while (0)

// a pair of CUDA events released on every exit path (the propagators throw on CUDA errors)
struct EventPair {
    cudaEvent_t a = nullptr, b = nullptr;
    EventPair() {
        CUDA_CHECK(cudaEventCreate(&a));
        if (cudaEventCreate(&b) != cudaSuccess) { cudaEventDestroy(a); a = nullptr; fail(PB200_ERR_CUDA, "cudaEventCreate failed"); }
    }
    ~EventPair() { if (a) cudaEventDestroy(a); if (b) cudaEventDestroy(b); }
    void start(cudaStream_t s) { CUDA_CHECK(cudaEventRecord(a, s)); }
    float stop_ms(cudaStream_t s) {   // device time since start(); waits for the stream's work so far
        CUDA_CHECK(cudaEventRecord(b, s));
        CUDA_CHECK(cudaEventSynchronize(b));
        float ms = 0.f;
        CUDA_CHECK(cudaEventElapsedTime(&ms, a, b));
        return ms;
    }
    EventPair(const EventPair&) = delete;
    EventPair& operator=(const EventPair&) = delete;
};

#define PB200_MAX_DEVICES 64

// NVTX range over a C-ABI entry point (visible in nsys / ncu timelines; a no-op without a profiler attached)
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
    NvtxRange(const NvtxRange&) = delete;
    NvtxRange& operator=(const NvtxRange&) = delete;
};

static int env_int(const char* name, int dflt) {
    const char* s = getenv(name);
    return s ? atoi(s) : dflt;
}

// ---- process-wide pool of device buffers ------------------------------------------------------------------
// A caller that builds one plan per Sequence (QutipEmulator.from_sequence(...).run(), bench.py's end-to-end leg,
// one plan per trajectory batch) would otherwise pay cudaMalloc / cudaFree (a device synchronisation each) for
// ~10 state-sized buffers per plan.  Freed buffers are kept per device, keyed by size, up to PB200_POOL_MIB
// (default 16 GiB); a plan synchronises its stream before returning buffers, so reuse by another plan is safe.
struct DevicePool {
    std::mutex mu;
    std::multimap<size_t, void*> free_list[PB200_MAX_DEVICES];
    std::unordered_map<void*, size_t> size_of;
    size_t held[PB200_MAX_DEVICES] = {0};
};
static DevicePool& pool() { static DevicePool* p = new DevicePool(); return *p; }  // never destroyed (CUDA teardown order)

static void* pool_alloc(int dev, size_t bytes) {
    if (bytes == 0) bytes = 16;
    bytes = (bytes + 255) & ~(size_t)255;
    DevicePool& pl = pool();
    if (dev >= 0 && dev < PB200_MAX_DEVICES) {
        std::lock_guard<std::mutex> lk(pl.mu);
        auto it = pl.free_list[dev].lower_bound(bytes);
        if (it != pl.free_list[dev].end() && it->first <= bytes + bytes / 4) {
            void* p = it->second;
            pl.held[dev] -= it->first;
            pl.free_list[dev].erase(it);
            return p;
        }
    }
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) {  // give the cached buffers back to the driver and retry once
        cudaGetLastError();
        {
            std::lock_guard<std::mutex> lk(pl.mu);
            if (dev >= 0 && dev < PB200_MAX_DEVICES) {
                for (auto& kv : pl.free_list[dev]) { pl.size_of.erase(kv.second); cudaFree(kv.second); }
                pl.free_list[dev].clear(); pl.held[dev] = 0;
            }
        }
        CUDA_CHECK(cudaMalloc(&p, bytes));
    }
    std::lock_guard<std::mutex> lk(pl.mu);
    pl.size_of[p] = bytes;
    return p;
}

static void pool_free(int dev, void* p) {
    if (!p) return;
    DevicePool& pl = pool();
    static const size_t cap = (size_t)std::max(0, env_int("PB200_POOL_MIB", 16384)) << 20;
    {
        std::lock_guard<std::mutex> lk(pl.mu);
        auto it = pl.size_of.find(p);
        if (it != pl.size_of.end() && dev >= 0 && dev < PB200_MAX_DEVICES && pl.held[dev] + it->second <= cap) {
            pl.free_list[dev].emplace(it->second, p);
            pl.held[dev] += it->second;
            return;
        }
        if (it != pl.size_of.end()) pl.size_of.erase(it);
    }
    cudaFree(p);
}

struct Plan;

// The one owner of a pool buffer, and the only caller of pool_alloc / pool_free.  The pool is not stream-ordered, so a
// buffer goes back only once the stream that uses it is idle: release (destructor, reset, move-assignment) synchronises
// the owning plan's `stream` field, read at that moment so that pb200_plan_set_stream is honoured.  Release also runs on
// error exits, so a failed synchronisation is cleared, never thrown.
template <typename T>
class DevBuf {
  public:
    DevBuf() = default;
    DevBuf(const Plan& P, size_t n) { reset(P, n); }
    DevBuf(DevBuf&& o) noexcept : dev_(o.dev_), stream_(o.stream_), n_(o.n_), p_(o.p_) { o.p_ = nullptr; o.n_ = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            release();
            dev_ = o.dev_; stream_ = o.stream_; n_ = o.n_; p_ = o.p_;
            o.p_ = nullptr; o.n_ = 0;
        }
        return *this;
    }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }

    // release the buffer, then take n elements on P's device, used by P's stream
    void reset(const Plan& P, size_t n);
    void release() noexcept {
        if (!p_) return;
        if (cudaStreamSynchronize(*stream_) != cudaSuccess) cudaGetLastError();
        pool_free(dev_, p_);
        p_ = nullptr; n_ = 0;
    }
    T* get() const { return p_; }
    size_t size() const { return n_; }
    explicit operator bool() const { return p_ != nullptr; }

  private:
    int dev_ = -1;
    const cudaStream_t* stream_ = nullptr;
    size_t n_ = 0;
    T* p_ = nullptr;
};

// tile of the Taylor stage kernel: 2^13 amplitudes (128 KiB), one CTA of 512 threads per SM, 16 amplitudes per thread.
// Measured on C2 (N = 20, H100): 44.1 us per order against 45.1 at 2^12 and 48.9 at 2^11, 42.9 with the evict-last
// store of chi_{k+1} (DESIGN.md section 8).
constexpr int kTaylorTileBits = 13;
constexpr int kTaylorRegBits = 4;
// complex-drive steps (stage_d2_taylor_kernel<..., CPLX = true>): the same tile, 256 threads of 32 amplitudes
constexpr int kTaylorCplxRegBits = 5;
// shared memory of the Taylor stage with several detuning shapes: the tile, the per-bit table, and the shapes' sums of
// every order's coefficients per register-bit pattern and per thread (stage_d2_taylor_kernel<..., PB200_TAYLOR_SMAX>)
static size_t taylor_shapes_smem(int n) {
    return ((size_t)16 << kTaylorTileBits) +
           (size_t)(taylor_table_stride(n, PB200_TAYLOR_SMAX) +
                    (PB200_TAYLOR_PMAX + 1) * ((1 << kTaylorRegBits) + (1 << (kTaylorTileBits - kTaylorRegBits)))) * 8;
}
// tile of the Chebyshev / Lanczos stage kernels (stage_d2_rb_kernel, stage_d2_fwd_kernel): 2^11 amplitudes, 8 per thread
constexpr int kStageTileBits = 11;
constexpr int kStageRegBits = 3;
// qubits above the tile that a pass still reaches by partner loads from global memory (plan_passes)
constexpr int kMaxExtraBits = 16;
// a state-vector shard holds 2^L amplitudes, 13 <= L <= 29: at least one tile, and the local bits above the tile
// (at most 16) stay partner loads of the single-pass geometry
constexpr int kShardMaxLocalBits = 29;
static_assert(kShardMaxLocalBits - kTaylorTileBits <= kMaxExtraBits, "a shard's local bits fit the single-pass geometry");

// Every instantiation of the tiled Taylor stage (stage_d2_taylor_kernel), keyed by its template flags: device_setup raises
// the shared-memory limit of each, launch_taylor_order launches the one a stage selects.  Shard variants launch without
// programmatic dependent launch, because their orders wait for their peers through events.
enum class TaylorSmem { Tile, TileTable, Shapes };   // the tile; + d2_table_stride(N) doubles; taylor_shapes_smem(N)
struct TaylorVariant {
    bool uniform, real_g, shard;
    int ns;
    bool cplx;
    void (*kernel)(TaylorArgs);
    int rb;
    TaylorSmem smem;
    bool pdl;
    bool diss = false;   // master equation (TaylorArgs::n_pair > 0)
    bool src32 = false, out32 = false;   // single-precision chi_k / chi_{k+1} and G_k (TaylorArgs::src32, out32)
};

static const std::vector<TaylorVariant>& taylor_variants() {
    constexpr int TB = kTaylorTileBits, RB = kTaylorRegBits, RBC = kTaylorCplxRegBits, SM = PB200_TAYLOR_SMAX;
    using S = TaylorSmem;
    static const std::vector<TaylorVariant> v = {
        // one state, one drive coefficient (C2, C5)
        {true,  true,  false, 0,  false, stage_d2_taylor_kernel<true, true, TB, RB, false, 0, false>,     RB,  S::Tile,      true},
        {true,  false, false, 0,  false, stage_d2_taylor_kernel<true, false, TB, RB, false, 0, false>,    RB,  S::TileTable, true},
        // ... the tail orders of their steps in single precision: the order at k_lo (fp64 -> fp32) and those after it
        {true,  true,  false, 0,  false, stage_d2_taylor_kernel<true, true, TB, RB, false, 0, false, false, false, true>,
         RB, S::Tile, true, false, false, true},
        {true,  true,  false, 0,  false, stage_d2_taylor_kernel<true, true, TB, RB, false, 0, false, false, true, true>,
         RB, S::Tile, true, false, true, true},
        {true,  false, false, 0,  false, stage_d2_taylor_kernel<true, false, TB, RB, false, 0, false, false, false, true>,
         RB, S::TileTable, true, false, false, true},
        {true,  false, false, 0,  false, stage_d2_taylor_kernel<true, false, TB, RB, false, 0, false, false, true, true>,
         RB, S::TileTable, true, false, true, true},
        // trajectory batch, per-qubit factors of one detuning shape (C4)
        {false, false, false, 1,  false, stage_d2_taylor_kernel<false, false, TB, RB, false, 1, false>,   RB,  S::TileTable, true},
        // several detuning shapes: one state (detuning maps), batches
        {true,  true,  false, SM, false, stage_d2_taylor_kernel<true, true, TB, RB, false, SM, false>,    RB,  S::Shapes,    true},
        {true,  false, false, SM, false, stage_d2_taylor_kernel<true, false, TB, RB, false, SM, false>,   RB,  S::Shapes,    true},
        {false, false, false, SM, false, stage_d2_taylor_kernel<false, false, TB, RB, false, SM, false>,  RB,  S::Shapes,    true},
        // state-vector shards
        {true,  true,  true,  0,  false, stage_d2_taylor_kernel<true, true, TB, RB, true, 0, false>,      RB,  S::Tile,      false},
        {true,  false, true,  0,  false, stage_d2_taylor_kernel<true, false, TB, RB, true, 0, false>,     RB,  S::TileTable, false},
        {true,  true,  true,  0,  false, stage_d2_taylor_kernel<true, true, TB, RB, true, 0, false, false, false, true>,
         RB, S::Tile, false, false, false, true},
        {true,  true,  true,  0,  false, stage_d2_taylor_kernel<true, true, TB, RB, true, 0, false, false, true, true>,
         RB, S::Tile, false, false, true, true},
        {true,  false, true,  0,  false, stage_d2_taylor_kernel<true, false, TB, RB, true, 0, false, false, false, true>,
         RB, S::TileTable, false, false, false, true},
        {true,  false, true,  0,  false, stage_d2_taylor_kernel<true, false, TB, RB, true, 0, false, false, true, true>,
         RB, S::TileTable, false, false, true, true},
        {true,  true,  true,  SM, false, stage_d2_taylor_kernel<true, true, TB, RB, true, SM, false>,     RB,  S::Shapes,    false},
        {true,  false, true,  SM, false, stage_d2_taylor_kernel<true, false, TB, RB, true, SM, false>,    RB,  S::Shapes,    false},
        // complex drive: the phase moves inside the step
        {true,  false, false, 0,  true,  stage_d2_taylor_kernel<true, false, TB, RBC, false, 0, true>,    RBC, S::TileTable, true},
        {false, false, false, 1,  true,  stage_d2_taylor_kernel<false, false, TB, RBC, false, 1, true>,   RBC, S::TileTable, true},
        {true,  false, false, SM, true,  stage_d2_taylor_kernel<true, false, TB, RBC, false, SM, true>,   RBC, S::Shapes,    true},
        {false, false, false, SM, true,  stage_d2_taylor_kernel<false, false, TB, RBC, false, SM, true>,  RBC, S::Shapes,    true},
        {true,  false, true,  0,  true,  stage_d2_taylor_kernel<true, false, TB, RBC, true, 0, true>,     RBC, S::TileTable, false},
        {true,  false, true,  SM, true,  stage_d2_taylor_kernel<true, false, TB, RBC, true, SM, true>,    RBC, S::Shapes,    false},
        // master equation on vec(rho): the batch gather (the column drive is -conj(omega)), one or several shapes
        {false, false, false, 1,  false, stage_d2_taylor_kernel<false, false, TB, RBC, false, 1, false, true>,  RBC, S::TileTable, true, true},
        {false, false, false, SM, false, stage_d2_taylor_kernel<false, false, TB, RBC, false, SM, false, true>, RBC, S::Shapes,    true, true},
        // ... under a drive whose phase moves inside the step (column bits: the signed sum changes sign)
        {false, false, false, 1,  true,  stage_d2_taylor_kernel<false, false, TB, RBC, false, 1, true, true>,   RBC, S::TileTable, true, true},
        {false, false, false, SM, true,  stage_d2_taylor_kernel<false, false, TB, RBC, false, SM, true, true>,  RBC, S::Shapes,    true, true},
        // ... split over state-vector shards by its top row bits
        {false, false, true,  1,  false, stage_d2_taylor_kernel<false, false, TB, RBC, true, 1, false, true>,   RBC, S::TileTable, false, true},
        {false, false, true,  SM, false, stage_d2_taylor_kernel<false, false, TB, RBC, true, SM, false, true>,  RBC, S::Shapes,    false, true},
    };
    return v;
}

// dynamic shared memory of a variant on N qubits: the tile, the interaction's factors and couplings (taylor_dint_setup), then the
// per-bit table or the shapes' sums
static size_t taylor_variant_smem(const TaylorVariant& v, int n) {
    const size_t tile = (size_t)16 << kTaylorTileBits;
    const size_t rest = v.smem == TaylorSmem::Shapes      ? taylor_shapes_smem(n) - tile
                        : v.smem == TaylorSmem::TileTable ? (size_t)d2_table_stride(n) * 8
                                                          : 0;
    return tile + (size_t)(taylor_dint_doubles(kTaylorTileBits, v.rb) + n * n) * 8 + rest;
}

// once per device and process: SM count, > 48 KB of dynamic shared memory for the tile kernels
static int device_setup(int dev) {
    static std::mutex mu;
    static int sm_count[PB200_MAX_DEVICES] = {0};
    std::lock_guard<std::mutex> lk(mu);
    if (dev >= 0 && dev < PB200_MAX_DEVICES && sm_count[dev] > 0) return sm_count[dev];
    int sms = 0;
    CUDA_CHECK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int max_smem = (1 << 13) * 16 + 1024;
    CUDA_CHECK(cudaFuncSetAttribute(stage_d2_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CUDA_CHECK(cudaFuncSetAttribute(stage_d2_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CUDA_CHECK(cudaFuncSetAttribute(stage_d2_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    constexpr int TB = kStageTileBits, RB = kStageRegBits;
    CUDA_CHECK(cudaFuncSetAttribute(stage_d2_rb_kernel<true, true, TB, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CUDA_CHECK(cudaFuncSetAttribute(stage_d2_rb_kernel<true, false, TB, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    CUDA_CHECK(cudaFuncSetAttribute(stage_d2_rb_kernel<false, false, TB, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    for (const TaylorVariant& v : taylor_variants())   // N <= 64
        CUDA_CHECK(cudaFuncSetAttribute(v.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)taylor_variant_smem(v, 64)));
    CUDA_CHECK(cudaFuncSetAttribute(stage_d2_fwd_kernel<true, TB, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 2048 * 16 + 256));
    CUDA_CHECK(cudaFuncSetAttribute(stage_d2_fwd_kernel<false, TB, RB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 2048 * 16 + 256));
    if (dev >= 0 && dev < PB200_MAX_DEVICES) sm_count[dev] = sms;
    return sms;
}

struct DriveTables {  // one (trajectory, drive): rows x interpolants
    std::vector<PiecewiseCubic<cplx>> coef;
    std::vector<PiecewiseCubic<double>> det;
    std::vector<double> coef_scale, det_scale;  // max |sample| per row
};

struct Plan {
    pb200_plan_desc desc;
    std::vector<double> times;
    int n = 0, dim = 0, B = 1;
    long long D = 0;
    int n_drives = 0;
    cudaStream_t stream = nullptr;
    // the stream the plan created (until pb200_plan_set_stream replaces it).  Declared before every DevBuf, so it is
    // destroyed after them: their release synchronises `stream`
    struct OwnedStream {
        cudaStream_t s = nullptr;
        OwnedStream() = default;
        OwnedStream(const OwnedStream&) = delete;
        OwnedStream& operator=(const OwnedStream&) = delete;
        ~OwnedStream() { reset(); }
        void reset() {
            if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); s = nullptr; }
        }
    } owned_stream;
    // device buffers
    DevBuf<c2> buf[3];
    DevBuf<c2> aux[6];  // [0..3] chain pools, [4..5] check copies
    int cur = 0;  // index of the current state buffer
    DevBuf<double> dint;
    DevBuf<double> cpl;      // the couplings behind dint, N x N per trajectory slot (TaylorArgs::cpl)
    bool dint_shared = true;
    bool has_interaction = false;
    DevBuf<double> d_table;  // per-exponential coefficient tables
    DevBuf<double> d_scratch;  // bins for reductions
    // host-side interpolants: [traj][drive]
    std::vector<std::vector<DriveTables>> tabs;
    std::vector<std::vector<bool>> tabs_set;
    // Dint bounds per |r>-count (shared-Dint case) and global bounds per trajectory
    std::vector<double> dmin_cnt, dmax_cnt;
    std::vector<double> dmin_traj, dmax_traj;
    bool state_set = false;
    int sm_count = 132;
    // Lindblad: per-qudit generators of the dissipator on the (row, column) digit pair
    std::vector<std::vector<cplx>> diss_gen;
    // Krylov (Lanczos) propagator workspace
    DevBuf<c2> kry; int kry_cap = 0;        // (kry_cap + 3) vectors of B*D
    DevBuf<double> d_kry;                   // alpha[m][B], beta[m][B], acc[3][B][2], norm[B], y[B][m][2]
    int m_last = 8;
    bool has_diss = false;
    // the dissipator as the Taylor stage applies it (TaylorArgs::dw, df), when it qualifies (diss_taylor_analyse)
    struct DissTaylor {
        bool ok = false;
        const char* why = "";
        c2 dw[4] = {}, df[4] = {};
        bool flip = false;        // some both-flip entry is non-zero
        double norm = 0.0;        // bound on the 2-norm of the dissipator (max row / column sum)
    } diss_tay;
    // Monte-Carlo wave function: single-qudit collapse operators (L^+L diagonal), thresholds, RNG
    std::vector<std::vector<cplx>> jump_ops;      // [n_ops][d*d]
    std::vector<std::vector<double>> jump_ldl;    // [n_ops][d]: diagonal of L^+L
    std::vector<std::vector<cplx>> jump_ldl_full; // [n_ops][d*d]: L^+L
    bool jump_diag = true;                        // every L^+L is diagonal (decay = one elementwise kernel)
    bool has_collapse = false;
    // XY mode: exchange couplings on the device, their absolute row sums (spectral bound)
    DevBuf<double> d_xy; bool xy_shared = true; bool has_xy = false; int xy_u = 0, xy_d = 1;
    std::vector<double> xy_norm;  // per trajectory: sum_{i<j} |Uxy_ij| (pairs not touching the SLM mask)
    // XY mode with an SLM mask: the interaction of the pairs touching a masked qudit is weighted by the
    // interpolated 0/1 coefficient slm_coef(t) (hamiltonian.py:399-424)
    bool has_slm = false; unsigned long long slm_bits = 0; PiecewiseCubic<double> slm_coef;
    DevBuf<double> dint2;                    // interaction diagonal of the pairs touching the mask
    std::vector<double> xy_norm2, dmin2_traj, dmax2_traj;
    std::mt19937_64 rng;
    std::vector<double> thresholds;               // per trajectory
    std::vector<long long> jump_count;
    // step-controller state kept between pb200_propagate calls (evaluation times cut a run into many calls):
    // interval classification of the sampling grid (cache key = window, rough_tol) and the current smooth-step length,
    // with the options it was reached under
    struct FineCache { bool valid = false; int window = -1; double rtol = -1.0; std::vector<char> fine, jump; std::vector<int> dist; } fine_cache;
    struct CtrlOptions {
        double gtol = 0.0; bool extrap = false; int order = 0, Kmax = 0;
        bool operator==(const CtrlOptions& o) const {
            return gtol == o.gtol && extrap == o.extrap && order == o.order && Kmax == o.Kmax;
        }
    };
    double ctrl_Kc = -1.0; CtrlOptions ctrl_opts; double ctrl_t_end = -1e300;
    // partner-sum forwarding between Clenshaw stages (stage_d2_fwd_kernel): one buffer of forwarded sums per chain
    DevBuf<c2> wbuf[2];
    // time-dependent Taylor propagator: the drive relative to the phase of its largest sample, half-width of H at the
    // sampling times, extra ring buffers (beyond buf / aux) for polynomial degrees > 2
    struct TaylorCache {
        bool valid = false, ok = false;
        const char* why = "";              // why not, once valid
        c2 unit{1.0, 0.0};                 // phase of the reference row's largest sample
        PiecewiseCubic<double> om;         // Re omega(t), omega = reference row x conj(unit)
        PiecewiseCubic<double> om_im;      // Im omega(t) (phase_moves only)
        bool phase_moves = false;          // omega is not real: the steps are classified (TaylorStep::drive)
        std::vector<double> w_knot;        // spectral half-width of H at the sampling times
        // separable per-(trajectory, qubit) drives: coef = a unit omega(t), det = theta(t) + sum_s c_s M_s(t)
        bool uniform = true;               // one state, one coefficient for every qubit (a = 1, c = 0)
        bool drive_uniform = true;         // one state, a = 1 (the detuning may have shapes)
        int ns = 0;                        // detuning shapes, <= PB200_TAYLOR_SMAX
        PiecewiseCubic<double> shape[PB200_TAYLOR_SMAX];   // M_s(t)
        std::vector<cplx> a;               // [B][N] per qubit
        // vec(rho) under a moving phase (taylor_prepare): the column qudits' factors are their rows' a, and the table
        // holds -conj(a unit) on the column bits, the drive -conj(unit omega) of any unit.  A constant phase keeps the
        // column factors of the fit (a_col unit = -conj(a_row unit) for the reference unit only)
        bool conj_cols = false;
        std::vector<double> c;             // [B][N][ns]
        double a_sum_max = 0.0;            // max over trajectories of sum_k |a|
        double c_sum_max[PB200_TAYLOR_SMAX] = {};   // max over trajectories of sum_k |c_s|
        // 0: [B][3N+2] device table of one shape (d2_table_stride); PB200_TAYLOR_SMAX: [B][taylor_table_stride(N, SMAX)]
        // (several shapes, or shapes on a uniform drive)
        int tab_shapes = 0;
        std::vector<double> tab_host;      // device table image with `unit`
        DevBuf<double> d_tab;
        c2 tab_unit{1.0, 0.0};             // the unit d_tab holds now (steps of one rotated phase upload their own)
    } tay;
    std::vector<DevBuf<c2>> tay_ws;
    // state-vector shard (pb200_plan_create_shard): the top shard_bits qubits of the global index equal `shard`; n is
    // the global N, D = 2^(N - shard_bits) the slice this plan holds.  `group` = every shard, by index, once linked
    int shard_bits = 0, shard = 0;
    std::vector<Plan*> group;
    long long shard_offset() const { return (long long)shard << (n - shard_bits); }
    bool all_uniform() const {
        for (int q = 0; q < n_drives; ++q)
            if (!desc.drives[q].uniform) return false;
        return true;
    }
};

template <typename T>
void DevBuf<T>::reset(const Plan& P, size_t n) {
    release();
    dev_ = P.desc.device;
    stream_ = &P.stream;
    p_ = static_cast<T*>(pool_alloc(dev_, sizeof(T) * n));
    n_ = n;
}

// device sums: zero acc[0, n), queue the reduction kernels (`launch`), then copy the sums to `host` and wait for them.
// sum_launch / sum_fetch split it where several streams reduce at once.
template <typename F>
static void sum_launch(const Plan& P, double* acc, size_t n, F&& launch) {
    CUDA_CHECK(cudaMemsetAsync(acc, 0, sizeof(double) * n, P.stream));
    launch();
    CUDA_CHECK(cudaGetLastError());
}

static void sum_fetch(const Plan& P, const double* acc, size_t n, double* host) {
    CUDA_CHECK(cudaMemcpyAsync(host, acc, sizeof(double) * n, cudaMemcpyDeviceToHost, P.stream));
    CUDA_CHECK(cudaStreamSynchronize(P.stream));
}

template <typename F>
static void device_sum(const Plan& P, double* acc, size_t n, double* host, F&& launch) {
    sum_launch(P, acc, n, launch);
    sum_fetch(P, acc, n, host);
}

// argument checks shared by the C-ABI entry points
static void check_traj_range(const Plan& P, int traj0, int count, const char* who) {
    if (traj0 < 0 || count < 1 || traj0 + count > P.B)
        fail(PB200_ERR_INVALID, "%s: trajectory range [%d, %d) outside [0, %d)", who, traj0, traj0 + count, P.B);
}

static void check_drives_set(const Plan& P, const char* who) {
    for (int tr = 0; tr < P.B; ++tr)
        for (int q = 0; q < P.n_drives; ++q)
            if (!P.tabs_set[tr][q]) fail(PB200_ERR_STATE, "%s: drive %d of trajectory %d not set", who, q, tr);
}

// launch with (optional) programmatic dependent launch: the kernel's prologue overlaps the tail of the
// previous stage kernel; the kernel itself executes griddepcontrol.wait before its first global read
template <typename... KArgs, typename... Args>
static void launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                     Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...));
}

// ---------------------------------------------------------------------------
static std::vector<PassGeom> plan_passes(int N, int TB, int EX) {
    std::vector<PassGeom> passes;
    PassGeom g{};
    g.n_bits = N;
    if (N <= TB) {
        g.lo_bits = N; g.hi_shift = N; g.hi_bits = 0;
        g.tile_flip_mask = (N >= 32) ? 0xffffffffu : ((1u << N) - 1u);
        g.extra_mask = 0; g.first_pass = 1;
        passes.push_back(g);
        return passes;
    }
    if (N - TB <= EX) {
        g.lo_bits = TB; g.hi_shift = TB; g.hi_bits = 0;
        g.tile_flip_mask = (1u << TB) - 1u;
        g.extra_mask = ((1ULL << N) - 1ULL) & ~((1ULL << TB) - 1ULL);
        g.first_pass = 1;
        passes.push_back(g);
        return passes;
    }
    // pass A: the TB low bits
    g.lo_bits = TB; g.hi_shift = TB; g.hi_bits = 0;
    g.tile_flip_mask = (1u << TB) - 1u; g.extra_mask = 0; g.first_pass = 1;
    passes.push_back(g);
    int next = TB;  // first bit not yet covered
    const int min_row_bits = 2;  // rows of >= 64 B
    while (next < N) {
        int rem = N - next;
        PassGeom p{};
        p.n_bits = N; p.first_pass = 0;
        int hb = std::min(rem, TB - min_row_bits);
        // leftover bits small enough -> take them as global-load extras
        int left = rem - hb;
        p.hi_bits = hb; p.hi_shift = next; p.lo_bits = TB - hb;
        p.tile_flip_mask = ((1u << hb) - 1u) << p.lo_bits;
        p.extra_mask = 0;
        if (left > 0 && left <= EX) {
            p.extra_mask = ((1ULL << N) - 1ULL) & ~((1ULL << (next + hb)) - 1ULL);
            left = 0;
            next = N;
        } else {
            next += hb;
        }
        passes.push_back(p);
    }
    return passes;
}

// ---------------------------------------------------------------------------
struct ExpParams {  // one exponential exp(-i G), G from Magnus moments
    // [traj][drive][row] unscaled g (complex) and theta; w common
    std::vector<cplx> g;
    std::vector<double> th;
    double w = 0.0;
    double wc = 0.0;  // weight of the SLM-masked pairs (XY mode with a mask); unused otherwise
};

static inline bool is_d2path(const Plan& P) { return P.dim == 2 && P.n_drives == 1 && !P.has_xy; }

// one state with one drive row: the stages read the drive from their arguments (UniformDrive), not from a table
static inline bool one_uniform_state(const Plan& P) { return is_d2path(P) && P.all_uniform() && P.B == 1; }

// what one propagate call decided for its exponentials
struct ExpChoice {
    bool krylov = false;            // Lanczos, else Chebyshev-Clenshaw
    bool fwd = false;               // partner-sum forwarding between Clenshaw stages (stage_d2_fwd_kernel)
    PassGeom fwd_passes[3];         // forwarding: a chain's first stage [0], the high-bit tile [1], later low-bit stages [2]
    std::vector<PassGeom> passes;   // stage geometry without forwarding
    bool dual_ok = false;           // two chains may share every launch
};

static inline size_t pidx(const Plan& P, int traj, int q, int row) {
    return ((size_t)traj * P.n_drives + q) * P.n + row;
}

struct StageIO {  // one Clenshaw stage of one chain
    const c2* v; const c2* psi; const c2* b2; c2* out;
    StageCoef coef; UniformDrive ud; const double* table; bool real_g;
    const double* beta_dev = nullptr;
    double* dot_acc = nullptr;  // fused <v,out>, <out,out> (only honoured by the register-blocked d=2 kernels)
    const LanczosFuse* lz = nullptr;  // fused Lanczos step (single-pass register-blocked geometry only)
    // partner-sum forwarding: 0 first stage of a chain (no forwarded input), 1 high-bit tile, 2 low-bit tile;
    // `emit`: a later stage of the chain consumes the sums of this stage's result
    int fwd_role = 0; bool fwd_emit = false; c2* wbuf = nullptr;
};

static StageArgs make_stage_args(const Plan& P, const PassGeom& geo, const StageIO& io, bool geo_is_last = true) {
    StageArgs a{};
    a.v = io.v; a.psi = io.psi; a.b2 = io.b2; a.out = io.out;
    a.dint = P.has_interaction ? P.dint.get() : nullptr;
    a.dint_stride = P.dint_shared ? 0 : P.D;
    a.D = P.D; a.geo = geo; a.coef = io.coef; a.u = io.ud; a.table = io.table;
    a.to_bit = P.desc.drives[0].state_to;
    a.from_is_one = P.desc.drives[0].state_from;
    a.beta_dev = io.beta_dev;
    a.dot_acc = (geo_is_last ? io.dot_acc : nullptr);
    if (geo_is_last && io.lz) a.lz = *io.lz;
    return a;
}

// d = 3 / 4 registers without an exchange term run on the register-blocked tiled kernel
static bool multilevel_eligible(const Plan& P) {
    return !P.has_xy && (P.dim == 3 || P.dim == 4) && P.n <= PB200_TILED_MAX_HIGH &&
           P.n >= (P.dim == 3 ? 2 : 1) && !(P.dim == 2);
}

static bool rb_eligible(const PassGeom& geo) {
    return geo.lo_bits + geo.hi_bits == kStageTileBits && (geo.first_pass || geo.hi_bits >= kStageRegBits);
}

// every pass of the geometry can carry two chains in one launch
static bool dual_chain_ok(const Plan& P, const std::vector<PassGeom>& passes) {
    if (!is_d2path(P)) return false;
    for (const PassGeom& g : passes)
        if (!rb_eligible(g)) return false;
    return (long long)P.B * 2 <= 65535;
}

// launch one stage for `n` (1 or 2) chains
static void launch_stage_multi(Plan& P, const std::vector<PassGeom>& passes, const StageIO* io, int n, bool uniform,
                               long long& launches) {
    const int N = P.n;
    if (is_d2path(P)) {
        bool real_g = true;
        for (int c = 0; c < n; ++c) real_g = real_g && io[c].real_g;
        for (size_t gi = 0; gi < passes.size(); ++gi) {
            const PassGeom& geo = passes[gi];
            const bool last_pass = (gi + 1 == passes.size());
            const int tbits = geo.lo_bits + geo.hi_bits;
            const long long tiles = P.D >> tbits;
            const int tsize = 1 << tbits;
            const size_t tab_bytes = uniform ? 0 : (size_t)d2_table_stride(N) * 8;
            if (rb_eligible(geo)) {
                constexpr int TB = kStageTileBits, RB = kStageRegBits;
                StageArgs2 m{};
                for (int c = 0; c < n; ++c) m.a[c] = make_stage_args(P, geo, io[c], last_pass);
                m.n_traj = P.B;
                dim3 grid((unsigned)tiles, (unsigned)(P.B * n)), block(tsize >> RB);
                const size_t smem = (size_t)tsize * 16 + tab_bytes;
                if (!uniform) launch_k(stage_d2_rb_kernel<false, false, TB, RB>, grid, block, smem, P.stream, true, m);
                else if (real_g) launch_k(stage_d2_rb_kernel<true, true, TB, RB>, grid, block, smem, P.stream, true, m);
                else launch_k(stage_d2_rb_kernel<true, false, TB, RB>, grid, block, smem, P.stream, true, m);
                ++launches;
            } else {
                for (int c = 0; c < n; ++c) {
                    StageArgs a = make_stage_args(P, geo, io[c]);
                    dim3 grid((unsigned)tiles, (unsigned)P.B);
                    int threads = std::min(256, std::max(32, tsize));
                    size_t smem = (size_t)tsize * 16 + tab_bytes;
                    if (uniform) {
                        if (real_g) stage_d2_kernel<true, true><<<grid, threads, smem, P.stream>>>(a);
                        else stage_d2_kernel<true, false><<<grid, threads, smem, P.stream>>>(a);
                    } else {
                        stage_d2_kernel<false, false><<<grid, threads, smem, P.stream>>>(a);
                    }
                    ++launches;
                }
            }
        }
    } else {
        for (int c = 0; c < n; ++c) {
            GenArgs a{};
            a.v = io[c].v; a.psi = io[c].psi; a.b2 = io[c].b2; a.out = io[c].out;
            a.dint = P.has_interaction ? P.dint.get() : nullptr;
            a.dint_stride = P.dint_shared ? 0 : P.D;
            a.D = P.D; a.n = N; a.dim = P.dim; a.n_drives = P.n_drives;
            for (int q = 0; q < P.n_drives; ++q) { a.to[q] = P.desc.drives[q].state_to; a.from[q] = P.desc.drives[q].state_from; }
            a.coef = io[c].coef; a.table = io[c].table; a.beta_dev = io[c].beta_dev;
            a.xy = P.has_xy ? P.d_xy.get() : nullptr; a.xy_stride = P.xy_shared ? 0 : (long long)N * N;
            a.xy_u = P.xy_u; a.xy_d = P.xy_d;
            a.slm_mask = P.has_slm ? P.slm_bits : 0ULL; a.dint2 = (P.has_slm && P.has_interaction) ? P.dint2.get() : nullptr;
            int threads = 256;
            if (multilevel_eligible(P)) {
                a.dot_acc = io[c].dot_acc;
                if (io[c].lz) a.lz = *io[c].lz;
                // register-blocked tiled kernel: 3^7 (9 amplitudes per thread) / 4^5 (4 per thread) amplitudes per CTA
                const int K = (P.dim == 3) ? 7 : 5;
                long long tsz = 1;
                for (int j = 0; j < std::min(K, N); ++j) tsz *= P.dim;
                dim3 tgrid((unsigned)(P.D / tsz), (unsigned)P.B);
                const size_t tsmem = (((size_t)tsz * 16 + 127) / 128) * 128 + (size_t)gen_table_stride(N, P.n_drives) * 8;
                if (P.dim == 3) stage_multilevel_rb_kernel<3, 7, 2><<<tgrid, threads, tsmem, P.stream>>>(a);
                else stage_multilevel_rb_kernel<4, 5, 1><<<tgrid, threads, tsmem, P.stream>>>(a);
                ++launches;
                continue;
            }
            long long blocks = std::min<long long>((P.D + threads - 1) / threads, (long long)P.sm_count * 8);
            dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)P.B);
            size_t smem = (size_t)gen_table_stride(N, P.n_drives) * 8 + (P.has_xy ? (size_t)N * N * 8 : 0);
            stage_generic_kernel<<<grid, threads, smem, P.stream>>>(a);
            ++launches;
        }
    }
}

// ---- partner-sum forwarding (uniform drives, Chebyshev chains) ----------------------------------------------------
// The second in-tile gather and the 64-byte rows of the high-bit tile cost as much shared-memory / LSU time as the
// forwarded sums save in L2 traffic once N >= 20, while at N = 18 (256-byte rows) forwarding saves L2 traffic
// without that penalty: it is used for the registers in between only (DESIGN.md section 6 gives both sides).
constexpr int kFwdMinN = 17, kFwdMaxN = 19;

static bool fwd_eligible(const Plan& P, const std::vector<PassGeom>& passes) {
    if (!one_uniform_state(P)) return false;
    if (passes.size() != 1 || passes[0].hi_bits != 0 || passes[0].lo_bits != kStageTileBits) return false;
    return P.n >= kFwdMinN && P.n <= kFwdMaxN;
}

static void plan_fwd_passes(const Plan& P, PassGeom geo[3]) {
    const int N = P.n, TB = kStageTileBits;
    const int hb = std::min(N - TB, TB - 2);
    const unsigned long long all = (N >= 64) ? ~0ULL : ((1ULL << N) - 1ULL);
    const unsigned long long rest = all & ~((1ULL << (TB + hb)) - 1ULL);
    PassGeom a{};
    a.n_bits = N; a.lo_bits = TB; a.hi_shift = TB; a.hi_bits = 0; a.first_pass = 1;
    a.tile_flip_mask = (1u << TB) - 1u;
    a.extra_mask = all & ~((1ULL << TB) - 1ULL);
    geo[0] = a;
    a.extra_mask = rest;
    geo[2] = a;
    PassGeom b{};
    b.n_bits = N; b.lo_bits = TB - hb; b.hi_shift = TB; b.hi_bits = hb; b.first_pass = 1;
    b.tile_flip_mask = ((1u << hb) - 1u) << b.lo_bits;
    b.extra_mask = rest;
    geo[1] = b;
}

// real_g: every chain's exponential is real (decided by run_chains before the chains emitted their stages)
static void launch_stage_fwd(Plan& P, const ExpChoice& X, const StageIO* io, int n, bool real_g, long long& launches) {
    constexpr int TB = kStageTileBits, RB = kStageRegBits;
    StageArgs2 m{};
    for (int c = 0; c < n; ++c) {
        StageArgs& a = m.a[c];
        a = make_stage_args(P, X.fwd_passes[io[c].fwd_role], io[c], true);
        a.w_in = (io[c].fwd_role > 0) ? io[c].wbuf : nullptr;
        a.w_out = io[c].fwd_emit ? io[c].wbuf : nullptr;
        a.w_plane = P.D * (long long)P.B;
    }
    m.n_traj = P.B;
    dim3 grid((unsigned)(P.D >> TB), (unsigned)(P.B * n));
    const size_t smem = (size_t)2 * ((size_t)16 << TB);
    if (real_g) launch_k(stage_d2_fwd_kernel<true, TB, RB>, grid, dim3(256), smem, P.stream, true, m);
    else launch_k(stage_d2_fwd_kernel<false, TB, RB>, grid, dim3(256), smem, P.stream, true, m);
    ++launches;
}

static void launch_stage(Plan& P, const std::vector<PassGeom>& passes, const c2* v, const c2* psi, const c2* b2,
                         c2* out, StageCoef coef, bool uniform, bool real_g, const UniformDrive& ud,
                         const double* table, long long& launches) {
    StageIO io{v, psi, b2, out, coef, ud, table, real_g, nullptr};
    launch_stage_multi(P, passes, &io, 1, uniform, launches);
}

// Fill the device-table entry (host staging) of one exponential for all
// trajectories; returns gamma0, rho (common to the batch).
static void build_tables(const Plan& P, const ExpParams& E, double& gamma0, double& rho, std::vector<double>& host,
                         bool d2path, bool scaled = true) {
    const int N = P.n, B = P.B, nd = P.n_drives;
    double lo = 1e300, hi = -1e300;
    for (int b = 0; b < B; ++b) {
        // drive norm bound
        double dr = 0.0;
        for (int q = 0; q < nd; ++q)
            for (int k = 0; k < N; ++k) dr += std::abs(E.g[pidx(P, b, q, k)]);
        if (P.has_xy) dr += std::fabs(E.w) * (P.xy_shared ? P.xy_norm[0] : P.xy_norm[b]);  // |flip-flop| <= 1
        if (P.has_xy && P.has_slm) dr += std::fabs(E.wc) * (P.xy_shared ? P.xy_norm2[0] : P.xy_norm2[b]);
        double dlo, dhi;
        const bool caseA = !P.has_slm && P.has_interaction && P.dint_shared && nd == 1 && P.desc.drives[0].uniform &&
                           P.desc.drives[0].state_from == P.desc.rydberg_state && !P.dmin_cnt.empty();
        if (caseA) {
            const double th = E.th[pidx(P, b, 0, 0)];
            dlo = 1e300; dhi = -1e300;
            for (int c = 0; c <= N; ++c) {
                if (P.dmin_cnt[c] > P.dmax_cnt[c]) continue;  // empty bin
                dlo = std::min(dlo, E.w * P.dmin_cnt[c] - th * c);
                dhi = std::max(dhi, E.w * P.dmax_cnt[c] - th * c);
            }
        } else {
            double dmn = 0.0, dmx = 0.0;
            if (P.has_interaction) {
                dmn = P.dint_shared ? P.dmin_traj[0] : P.dmin_traj[b];
                dmx = P.dint_shared ? P.dmax_traj[0] : P.dmax_traj[b];
            }
            dlo = E.w * dmn; dhi = E.w * dmx;
            if (P.has_slm && P.has_interaction) {  // second diagonal, weight wc (may be slightly outside [0, w])
                const double m2 = P.dint_shared ? P.dmin2_traj[0] : P.dmin2_traj[b];
                const double x2 = P.dint_shared ? P.dmax2_traj[0] : P.dmax2_traj[b];
                dlo += std::min(E.wc * m2, E.wc * x2); dhi += std::max(E.wc * m2, E.wc * x2);
            }
            for (int k = 0; k < N; ++k) {
                double mn = 0.0, mx = 0.0;  // a digit that is nobody's `from`
                for (int dgt = 0; dgt < P.dim; ++dgt) {
                    double val = 0.0;
                    for (int q = 0; q < nd; ++q)
                        if (P.desc.drives[q].state_from == dgt) val -= E.th[pidx(P, b, q, k)];
                    mn = std::min(mn, val); mx = std::max(mx, val);
                }
                // if every digit is some drive's `from`, 0 is not attainable; keeping it only widens the bound
                dlo += mn; dhi += mx;
            }
        }
        lo = std::min(lo, dlo - dr);
        hi = std::max(hi, dhi + dr);
    }
    gamma0 = 0.5 * (lo + hi);
    rho = std::max(0.5 * (hi - lo) * (1.0 + 1e-9), 1e-9);
    const double rho_bound = rho;
    if (!scaled) { gamma0 = 0.0; rho = 1.0; }  // raw operator (Krylov path); the bound is still reported
    const double inv = 1.0 / rho;
    if (d2path) {
        const int stride = d2_table_stride(N);
        host.assign((size_t)B * stride, 0.0);
        for (int b = 0; b < B; ++b) {
            double* t = host.data() + (size_t)b * stride;
            for (int k = 0; k < N; ++k) {
                const int p = N - 1 - k;  // bit position of qubit k
                const cplx g = E.g[pidx(P, b, 0, k)] * inv;
                t[2 * p] = g.real(); t[2 * p + 1] = g.imag();
                t[2 * N + p] = E.th[pidx(P, b, 0, k)] * inv;
            }
            t[3 * N] = E.w * inv; t[3 * N + 1] = gamma0 * inv;
        }
    } else {
        const int stride = gen_table_stride(N, nd);
        host.assign((size_t)B * stride, 0.0);
        for (int b = 0; b < B; ++b) {
            double* t = host.data() + (size_t)b * stride;
            for (int q = 0; q < nd; ++q) {
                double* tq = t + (size_t)q * 3 * N;
                for (int k = 0; k < N; ++k) {
                    const cplx g = E.g[pidx(P, b, q, k)] * inv;
                    tq[2 * k] = g.real(); tq[2 * k + 1] = g.imag();
                    tq[2 * N + k] = E.th[pidx(P, b, q, k)] * inv;
                }
            }
            t[stride - 3] = E.wc * inv; t[stride - 2] = E.w * inv; t[stride - 1] = gamma0 * inv;
        }
    }
    if (!scaled) rho = rho_bound;
}

struct Program {  // a batch of exponentials prepared on the host
    std::vector<double> tables;        // concatenated per-exponential tables
    std::vector<size_t> offset;        // start of each exponential's table
    std::vector<double> gamma0, rho;
    std::vector<std::vector<cplx>> cheb;
    std::vector<UniformDrive> ud;
    std::vector<char> real_g;
    // Lindblad splitting: dissipator exp(h D) applied before / after exponential e (0 = none)
    std::vector<double> pre_diss, post_diss;
    std::vector<ExpParams> raw;  // unscaled generators (Krylov path)
    std::vector<double> ktol;    // convergence tolerance of each Krylov exponential
};

static void ensure_table_capacity(Plan& P, size_t doubles) {
    if (doubles <= P.d_table.size()) return;
    P.d_table.reset(P, std::max(doubles, (size_t)1 << 16));
}

// One chain = a program (sequence of exponentials) applied to a state with its own buffers.  `next` emits
// the next Clenshaw stage; chains are independent, so two of them can share every kernel launch.
struct Chain {
    const Program* prog = nullptr;
    size_t table_base = 0;   // offset of this program's tables in P.d_table
    c2* psi = nullptr;       // input of the current exponential (never written by it)
    c2* pool[3] = {nullptr, nullptr, nullptr};  // private buffers
    bool psi_is_private = false;
    // exponential / Clenshaw state
    size_t e = 0; int j = -1;
    const c2* b1_buf = nullptr; cplx b1_scale = 0.0;
    int b2_kind = 0; c2* b2_buf = nullptr; cplx kappa = 0.0;
    c2* out = nullptr;
    c2* scratch[2] = {nullptr, nullptr};
    long long applies = 0; double max_rho = 0.0;
    int fwd_parity = 0; bool fwd_valid = false;   // partner-sum forwarding: geometry of the next stage, sums available
    bool fwd_q = false;                           // the forwarded sums include the Q plane (a complex launch wrote them)

    bool done() const { return e >= prog->cheb.size(); }
    c2* result() const { return psi; }

    void begin_exponential() {
        const std::vector<cplx>& a = prog->cheb[e];
        const int m = (int)a.size() - 1;
        j = m - 1;
        b1_buf = psi; b1_scale = a[m];
        b2_kind = 0; b2_buf = nullptr; kappa = 0.0; out = nullptr;
        // scratch: the two private buffers that are not the input
        int k = 0;
        for (int i = 0; i < 3 && k < 2; ++i)
            if (pool[i] != psi) scratch[k++] = pool[i];
    }
    bool next_real_g() const { return prog->real_g[e] != 0; }
    // fill io for the next stage and advance; requires !done().  `launch_real`: the stage runs in a launch of the real
    // forwarding kernel, which writes and reads only the P plane of the forwarded sums
    void next(const Plan& P, bool uniform, bool launch_real, StageIO& io) {
        if (j < 0) begin_exponential();
        const std::vector<cplx>& a = prog->cheb[e];
        const cplx ph = std::exp(cplx(0.0, -prog->gamma0[e]));
        const double factor = (j == 0) ? 1.0 : 2.0;
        const cplx phase = (j == 0) ? ph : cplx(1.0, 0.0);
        const cplx cg = phase * factor * b1_scale;
        const cplx cpsi = phase * (a[j] - (b2_kind == 2 ? kappa : cplx(0.0)));
        const cplx cb2 = (b2_kind == 1) ? -phase : cplx(0.0);
        if (b2_kind == 1) out = b2_buf;
        else out = (scratch[0] != b1_buf) ? scratch[0] : scratch[1];
        io.v = b1_buf; io.psi = psi; io.b2 = (b2_kind == 1) ? b2_buf : nullptr; io.out = out;
        io.coef = StageCoef{{cpsi.real(), cpsi.imag()}, {cb2.real(), cb2.imag()}, {cg.real(), cg.imag()}};
        io.ud = prog->ud[e];
        io.table = uniform ? nullptr : P.d_table.get() + table_base + prog->offset[e];
        io.real_g = prog->real_g[e] != 0;
        // partner-sum forwarding: this stage's geometry and whether a later stage of the chain consumes its sums.  A
        // complex launch also reads the Q plane, which a real launch does not write: after a real launch the first
        // complex stage gathers all its partners itself, as the first stage of a chain does
        if (!launch_real && !fwd_q) fwd_valid = false;
        io.fwd_role = !fwd_valid ? 0 : (fwd_parity ? 1 : 2);
        io.fwd_emit = !(j == 0 && e + 1 == prog->cheb.size());
        fwd_parity = (io.fwd_role == 1) ? 0 : 1;
        fwd_valid = io.fwd_emit;
        fwd_q = !launch_real;
        // shift the recurrence
        if (b1_buf == psi) { b2_kind = 2; kappa = b1_scale; b2_buf = nullptr; }
        else { b2_kind = 1; b2_buf = const_cast<c2*>(b1_buf); }
        b1_buf = out; b1_scale = 1.0;
        if (--j < 0) {  // exponential finished: its result becomes the next input
            applies += (long long)a.size() - 1;
            max_rho = std::max(max_rho, prog->rho[e]);
            if (!psi_is_private) {
                // the shared input stays untouched; the third private buffer joins the rotation
                psi_is_private = true;
            }
            psi = out;
            ++e;
        }
    }
};

static void apply_dissipator(Plan& P, c2* buf, double h, long long& launches);

static void run_chains(Plan& P, Chain* chains, int n, const ExpChoice& X, pb200_run_stats& st) {
    const bool uniform = one_uniform_state(P);
    if (!uniform) {
        size_t total = 0;
        for (int c = 0; c < n; ++c) { chains[c].table_base = total; total += chains[c].prog->tables.size(); }
        ensure_table_capacity(P, total);
        for (int c = 0; c < n; ++c)
            if (!chains[c].prog->tables.empty())
                CUDA_CHECK(cudaMemcpyAsync(P.d_table.get() + chains[c].table_base, chains[c].prog->tables.data(),
                                           chains[c].prog->tables.size() * sizeof(double), cudaMemcpyHostToDevice,
                                           P.stream));
    }
    long long launches = 0;
    StageIO io[2];
    if (X.fwd)
        for (int c = 0; c < n; ++c)
            if (!P.wbuf[c]) P.wbuf[c].reset(P, (size_t)P.D * P.B * 2);
    if (P.has_diss && n != 1) fail(PB200_ERR_STATE, "internal: Lindblad splitting runs one chain at a time");
    // PB200_MAGNUS_LOG: one line per forwarding stage and chain (what kernel and which forwarded sums it used)
    const bool log_fwd = X.fwd && env_int("PB200_MAGNUS_LOG", 0) != 0;
    if (log_fwd) fprintf(stderr, "magnus fwd chains=%d\n", n);
    while (true) {
        int k = 0;
        size_t e_before = 0;
        bool real_g = true;   // the stages of this launch all belong to real exponentials
        for (int c = 0; c < n; ++c)
            if (!chains[c].done()) real_g = real_g && chains[c].next_real_g();
        for (int c = 0; c < n; ++c)
            if (!chains[c].done()) {
                if (P.has_diss) {
                    e_before = chains[c].e;
                    if (chains[c].j < 0 && chains[c].prog->pre_diss[e_before] > 0.0)
                        apply_dissipator(P, chains[c].psi, chains[c].prog->pre_diss[e_before], launches);
                }
                io[k].wbuf = P.wbuf[c].get();
                chains[c].next(P, uniform, real_g, io[k]);
                if (log_fwd)
                    fprintf(stderr, "magnus fwd stage chain=%d exp_real=%d launch_real=%d role=%d\n", c,
                            (int)io[k].real_g, (int)real_g, io[k].fwd_role);
                ++k;
            }
        if (k == 0) break;
        if (X.fwd) launch_stage_fwd(P, X, io, k, real_g, launches);
        else launch_stage_multi(P, X.passes, io, k, uniform, launches);
        if (P.has_diss && chains[0].e != e_before && chains[0].prog->post_diss[e_before] > 0.0)
            apply_dissipator(P, chains[0].psi, chains[0].prog->post_diss[e_before], launches);
    }
    CUDA_CHECK(cudaGetLastError());
    st.n_launches += launches;
    for (int c = 0; c < n; ++c) {
        st.n_applies += chains[c].applies;
        st.max_rho = std::max(st.max_rho, chains[c].max_rho);
        st.n_exponentials += (long long)chains[c].prog->cheb.size();
    }
}

// eigen-decomposition of a real symmetric tridiagonal matrix (implicit QL, eigenvectors accumulated);
// d: diagonal (in) / eigenvalues (out), e: sub-diagonal e[0..n-2], z: n x n row-major, identity on entry
static void tridiag_ql(std::vector<double>& d, std::vector<double> e, std::vector<double>& z, int n) {
    e.resize(n, 0.0);
    for (int l = 0; l < n; ++l) {
        int iter = 0, m;
        do {
            for (m = l; m < n - 1; ++m) {
                const double dd = std::fabs(d[m]) + std::fabs(d[m + 1]);
                if (std::fabs(e[m]) <= 1e-300 + 2.3e-16 * dd) break;
            }
            if (m != l) {
                if (++iter > 200) break;
                double g = (d[l + 1] - d[l]) / (2.0 * e[l]);
                double r = std::hypot(g, 1.0);
                g = d[m] - d[l] + e[l] / (g + (g >= 0 ? std::fabs(r) : -std::fabs(r)));
                double s = 1.0, c = 1.0, p = 0.0;
                int i;
                for (i = m - 1; i >= l; --i) {
                    double f = s * e[i], b = c * e[i];
                    r = std::hypot(f, g);
                    e[i + 1] = r;
                    if (r == 0.0) { d[i + 1] -= p; e[m] = 0.0; break; }
                    s = f / r; c = g / r;
                    g = d[i + 1] - p;
                    r = (d[i] - g) * s + 2.0 * c * b;
                    p = s * r;
                    d[i + 1] = g + p;
                    g = c * r - b;
                    for (int k = 0; k < n; ++k) {
                        f = z[k * n + i + 1];
                        z[k * n + i + 1] = s * z[k * n + i] + c * f;
                        z[k * n + i] = c * z[k * n + i] - s * f;
                    }
                }
                if (r == 0.0 && i >= l) continue;
                d[l] -= p; e[l] = g; e[m] = 0.0;
            }
        } while (m != l);
    }
}

// y = exp(-i T_m) e_1 for the Lanczos tridiagonal T_m
static std::vector<cplx> tridiag_exp_e1(const double* alpha, const double* beta, int m) {
    std::vector<double> d(alpha, alpha + m), e(m > 1 ? m - 1 : 0), z((size_t)m * m, 0.0);
    for (int i = 0; i + 1 < m; ++i) e[i] = beta[i];
    for (int i = 0; i < m; ++i) z[(size_t)i * m + i] = 1.0;
    tridiag_ql(d, e, z, m);
    std::vector<cplx> y(m, cplx(0));
    for (int k = 0; k < m; ++k) {
        const cplx ph = std::exp(cplx(0.0, -d[k])) * z[k];  // z[0*m + k]: first component of eigenvector k
        for (int i = 0; i < m; ++i) y[i] += ph * z[(size_t)i * m + k];
    }
    return y;
}

static void ensure_krylov(Plan& P, int m_cap) {
    if (P.kry && P.kry_cap >= m_cap) return;
    P.kry.release(); P.d_kry.release();
    // basis vectors V_0 .. V_{m_cap} and the two raw vectors of the fused recurrence
    P.kry.reset(P, (size_t)P.D * P.B * (m_cap + 3));
    P.d_kry.reset(P, (size_t)m_cap * P.B * 2 + (size_t)6 * P.B + P.B + (size_t)P.B * m_cap * 2);
    P.kry_cap = m_cap;
}

// Largest Krylov dimension whose workspace fits: a third of the free device memory
static int krylov_capacity(const Plan& P) {
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) { cudaGetLastError(); return 64; }
    const double per_vec = (double)sizeof(c2) * (double)P.D * P.B;
    const int fit = (int)std::floor((double)free_b / 3.0 / per_vec) - 3;
    return std::max(8, std::min(64, fit));
}

// psi <- exp(-iG) psi by the Lanczos process: orthonormal basis V_0..V_{m-1} of the Krylov space of (G, psi),
// exponential of the m x m tridiagonal on the host, a-posteriori error estimate beta_{m-1} |y_{m-1}|.
// On the register-blocked kernels every iteration is ONE launch: the stage computes the raw vector
// r_j = G v_j - beta_{j-1} v_{j-1} with its two inner products fused, and the normalisation / orthogonalisation
// of v_{j+1} is folded into the own-element operands of the next stage (LanczosFuse, kernels.cuh).
static void krylov_exponential(Plan& P, const ExpParams& E, double tol, const ExpChoice& X, pb200_run_stats& st) {
    const std::vector<PassGeom>& passes = X.passes;
    if (P.kry_cap == 0) ensure_krylov(P, krylov_capacity(P));
    const int M = P.kry_cap;
    const int B = P.B;
    const long long D = P.D;
    const long long vstride = D * (long long)B;
    double* d_alpha = P.d_kry.get();
    double* d_beta = d_alpha + (size_t)M * B;
    double* d_acc = d_beta + (size_t)M * B;   // [3][B][2]
    double* d_norm = d_acc + (size_t)6 * B;
    double* d_y = d_norm + B;
    const bool d2path = is_d2path(P);
    const bool uniform = one_uniform_state(P);
    double gm, rh; std::vector<double> host;
    build_tables(P, E, gm, rh, host, d2path, /*scaled=*/false);
    st.max_rho = std::max(st.max_rho, rh);
    if (!uniform) {
        ensure_table_capacity(P, host.size());
        CUDA_CHECK(cudaMemcpyAsync(P.d_table.get(), host.data(), host.size() * sizeof(double), cudaMemcpyHostToDevice, P.stream));
    }
    UniformDrive ud{};
    ud.g = {E.g[0].real(), E.g[0].imag()}; ud.theta = E.th[0]; ud.w = E.w; ud.gamma = 0.0;
    const bool real_g = E.g[0].imag() == 0.0;
    bool fused_dot = d2path;
    for (const PassGeom& g : passes) fused_dot = fused_dot && rb_eligible(g);
    // one launch per iteration: single-pass register-blocked d = 2 geometry, or the tiled d = 3 / 4 kernel
    const bool fused = (fused_dot && passes.size() == 1) || (!d2path && multilevel_eligible(P));
    if (fused) fused_dot = true;
    c2* psi = P.buf[P.cur].get();
    c2* outb = P.buf[(P.cur + 1) % 3].get();
    c2* V = P.kry.get();                            // V_j = V + j * vstride
    c2* Rw[2] = {V + (size_t)(M + 1) * vstride, V + (size_t)(M + 2) * vstride};
    auto acc = [&](int j) { return d_acc + (size_t)(((j % 3) + 3) % 3) * 2 * B; };
    const long long rblocks = std::min<long long>((D + 255) / 256, (long long)P.sm_count * 4);
    dim3 rgrid((unsigned)std::max<long long>(rblocks, 1), (unsigned)B);
    long long launches = 0;
    CUDA_CHECK(cudaMemsetAsync(d_acc, 0, sizeof(double) * 6 * B, P.stream));
    dot2_kernel<<<rgrid, 256, 0, P.stream>>>(psi, psi, D, acc(2));
    normalize_copy_kernel<<<rgrid, 256, 0, P.stream>>>(V, psi, D, acc(2), d_norm, acc(1));
    launches += 2;
    int m_check = std::min(M, std::max(3, P.m_last));
    std::vector<double> ha((size_t)M * B), hb((size_t)M * B), hn(B), hacc((size_t)2 * B);
    std::vector<std::vector<cplx>> ys(B);
    int m_used = 0;
    int j = 0;
    while (true) {
        for (; j < m_check; ++j) {
            StageIO io{};
            io.coef = StageCoef{{0, 0}, {0, 0}, {1, 0}};
            io.ud = ud; io.table = uniform ? nullptr : P.d_table.get(); io.real_g = real_g;
            LanczosFuse lz{};
            if (fused) {
                // stage j: raw r_j from raw r_{j-1} (j >= 1) or from v_0 (j = 0); materialises v_j
                io.v = (j == 0) ? V : Rw[(j - 1) & 1];
                io.out = Rw[j & 1];
                io.dot_acc = acc(j);
                if (j >= 1) {
                    lz.vj = V + (size_t)(j - 1) * vstride;
                    lz.vjm1 = (j >= 2) ? V + (size_t)(j - 2) * vstride : nullptr;
                    lz.vout = V + (size_t)j * vstride;
                    lz.acc_prev = acc(j - 1);
                    lz.beta_prev = (j >= 2) ? d_beta + (size_t)(j - 2) * B : nullptr;
                    lz.alpha_out = d_alpha + (size_t)(j - 1) * B;
                    lz.beta_out = d_beta + (size_t)(j - 1) * B;
                    lz.acc_clear = acc(j + 1);
                    io.lz = &lz;
                }
                launch_stage_multi(P, passes, &io, 1, uniform, launches);
            } else {
                io.v = V + (size_t)j * vstride;
                io.b2 = (j > 0) ? V + (size_t)(j - 1) * vstride : nullptr;
                io.out = V + (size_t)(j + 1) * vstride;
                io.beta_dev = (j > 0) ? d_beta + (size_t)(j - 1) * B : nullptr;
                io.dot_acc = fused_dot ? acc(j) : nullptr;
                launch_stage_multi(P, passes, &io, 1, uniform, launches);
                if (!fused_dot) { dot2_kernel<<<rgrid, 256, 0, P.stream>>>(io.v, io.out, D, acc(j)); ++launches; }
                lanczos_update_kernel<<<rgrid, 256, 0, P.stream>>>(io.out, io.v, D, acc(j), d_alpha + (size_t)j * B,
                                                                   d_beta + (size_t)j * B, acc(j + 1));
                launches += 1;
            }
        }
        CUDA_CHECK(cudaGetLastError());
        const int n_rec = fused ? m_check - 1 : m_check;   // coefficients recorded on the device so far
        if (n_rec > 0) {
            CUDA_CHECK(cudaMemcpyAsync(ha.data(), d_alpha, sizeof(double) * (size_t)n_rec * B, cudaMemcpyDeviceToHost, P.stream));
            CUDA_CHECK(cudaMemcpyAsync(hb.data(), d_beta, sizeof(double) * (size_t)n_rec * B, cudaMemcpyDeviceToHost, P.stream));
        }
        if (fused) CUDA_CHECK(cudaMemcpyAsync(hacc.data(), acc(m_check - 1), sizeof(double) * 2 * B, cudaMemcpyDeviceToHost, P.stream));
        CUDA_CHECK(cudaMemcpyAsync(hn.data(), d_norm, sizeof(double) * B, cudaMemcpyDeviceToHost, P.stream));
        CUDA_CHECK(cudaStreamSynchronize(P.stream));
        if (fused)   // the last pair comes from the reductions of the last stage (the next stage would record it)
            for (int b = 0; b < B; ++b) {
                const double al = hacc[2 * b], ww = hacc[2 * b + 1], b2 = ww - al * al;
                ha[(size_t)(m_check - 1) * B + b] = al;
                hb[(size_t)(m_check - 1) * B + b] = (b2 > 1e-28 * std::max(ww, 1e-300)) ? std::sqrt(b2) : 0.0;
            }
        double worst = 0.0;
        for (int b = 0; b < B; ++b) {
            // per-trajectory effective dimension: stop at a breakdown (beta = 0: invariant subspace reached)
            int m = m_check;
            std::vector<double> al(m), be(m);
            for (int i = 0; i < m; ++i) { al[i] = ha[(size_t)i * B + b]; be[i] = hb[(size_t)i * B + b]; }
            for (int i = 0; i < m; ++i)
                if (be[i] == 0.0) { m = i + 1; break; }
            ys[b] = tridiag_exp_e1(al.data(), be.data(), m);
            const double err = (m < m_check || be[m - 1] == 0.0) ? 0.0 : hn[b] * be[m - 1] * std::abs(ys[b][m - 1]);
            worst = std::max(worst, err);
            ys[b].resize(m_check, cplx(0));
            for (cplx& z : ys[b]) z *= hn[b];
        }
        m_used = m_check;
        if (worst <= tol || m_check >= M) break;
        m_check = std::min(M, m_check + 4);
    }
    P.m_last = std::max(3, m_used - 1);
    std::vector<double> hy((size_t)B * m_used * 2);
    for (int b = 0; b < B; ++b)
        for (int i = 0; i < m_used; ++i) { hy[((size_t)b * m_used + i) * 2] = ys[b][i].real(); hy[((size_t)b * m_used + i) * 2 + 1] = ys[b][i].imag(); }
    CUDA_CHECK(cudaMemcpyAsync(d_y, hy.data(), sizeof(double) * hy.size(), cudaMemcpyHostToDevice, P.stream));
    krylov_combine_kernel<<<rgrid, 256, 0, P.stream>>>(outb, V, vstride, D, d_y, m_used);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaStreamSynchronize(P.stream));  // hy / host tables go out of scope
    launches += 1;
    P.cur = (P.cur + 1) % 3;
    st.n_launches += launches;
    st.n_applies += m_used;
    st.n_exponentials += 1;
}

static void run_program_krylov(Plan& P, const Program& prog, const ExpChoice& X, pb200_run_stats& st) {
    long long launches = 0;
    for (size_t e = 0; e < prog.raw.size(); ++e) {
        if (P.has_diss && prog.pre_diss[e] > 0.0) apply_dissipator(P, P.buf[P.cur].get(), prog.pre_diss[e], launches);
        krylov_exponential(P, prog.raw[e], prog.ktol.empty() ? 1e-12 : prog.ktol[e], X, st);
        if (P.has_diss && prog.post_diss[e] > 0.0) apply_dissipator(P, P.buf[P.cur].get(), prog.post_diss[e], launches);
    }
    st.n_launches += launches;
}

// apply exp(-iG) for every exponential in the program, in order, to the current state
static void run_program(Plan& P, const Program& prog, const ExpChoice& X, pb200_run_stats& st) {
    if (prog.cheb.empty()) return;
    if (X.krylov) { run_program_krylov(P, prog, X, st); return; }
    Chain ch;
    ch.prog = &prog;
    ch.psi = P.buf[P.cur].get();
    ch.psi_is_private = true;
    for (int i = 0; i < 3; ++i) ch.pool[i] = P.buf[i].get();
    run_chains(P, &ch, 1, X, st);
    for (int i = 0; i < 3; ++i)
        if (P.buf[i].get() == ch.result()) P.cur = i;
}

// ---------------------------------------------------------------------------
// the generator of the order-2 Magnus exponential over [a, b], m0 = int H dt (wc: the SLM weight), and on request the
// first moment m1 = (1/(b-a)) int (t - mid) H dt (m1->w = 0: the interaction strength is constant)
static ExpParams step_generator(const Plan& P, double a, double b, ExpParams* m1_out = nullptr) {
    const int N = P.n, B = P.B, nd = P.n_drives;
    ExpParams m0, m1;
    std::vector<cplx>& g0 = m0.g; std::vector<cplx>& g1 = m1.g;
    std::vector<double>& t0 = m0.th; std::vector<double>& t1 = m1.th;
    g0.assign((size_t)B * nd * N, cplx(0)); g1 = g0;
    t0.assign((size_t)B * nd * N, 0.0); t1 = t0;
    m0.w = b - a;
    if (P.has_slm) magnus_moments(P.slm_coef, P.times, a, b, m0.wc, m1.wc);
    for (int tr = 0; tr < B; ++tr)
        for (int q = 0; q < nd; ++q) {
            const DriveTables& T = P.tabs[tr][q];
            const int rows = (int)T.coef.size();
            for (int r = 0; r < rows; ++r) {
                cplx c0, c1; double d0, d1;
                magnus_moments(T.coef[r], P.times, a, b, c0, c1);
                magnus_moments(T.det[r], P.times, a, b, d0, d1);
                if (rows == 1) {
                    for (int k = 0; k < N; ++k) {
                        g0[pidx(P, tr, q, k)] = c0; g1[pidx(P, tr, q, k)] = c1;
                        t0[pidx(P, tr, q, k)] = d0; t1[pidx(P, tr, q, k)] = d1;
                    }
                } else {
                    g0[pidx(P, tr, q, r)] = c0; g1[pidx(P, tr, q, r)] = c1;
                    t0[pidx(P, tr, q, r)] = d0; t1[pidx(P, tr, q, r)] = d1;
                }
            }
        }
    if (m1_out) *m1_out = std::move(m1);
    return m0;
}

// spectral half-width of a generator
static double generator_rho(const Plan& P, const ExpParams& E) {
    double gamma0, rho; std::vector<double> scratch_tab;
    build_tables(P, E, gamma0, rho, scratch_tab, is_d2path(P));
    return rho;
}

static void add_exponential(const Plan& P, Program& prog, const ExpParams& E, double tol, const ExpChoice& X) {
    const bool d2path = is_d2path(P);
    double gamma0, rho;
    std::vector<double> host;
    build_tables(P, E, gamma0, rho, host, d2path);
    prog.offset.push_back(prog.tables.size());
    prog.tables.insert(prog.tables.end(), host.begin(), host.end());
    prog.gamma0.push_back(gamma0);
    prog.rho.push_back(rho);
    prog.cheb.push_back(chebyshev_exp_coeffs(rho, tol));
    UniformDrive ud{};
    const cplx g = E.g[0] / rho;
    ud.g = {g.real(), g.imag()};
    ud.theta = E.th[0] / rho; ud.w = E.w / rho; ud.gamma = gamma0 / rho;
    ud.to_bit = P.desc.drives[0].state_to;
    prog.ud.push_back(ud);
    prog.real_g.push_back(g.imag() == 0.0 ? 1 : 0);
    prog.pre_diss.push_back(0.0);
    prog.post_diss.push_back(0.0);
    if (X.krylov) { prog.raw.push_back(E); prog.ktol.push_back(tol); }
}

// exp(h*A) of a small dense matrix (scaling and squaring, Taylor order 20)
static std::vector<cplx> small_expm(const std::vector<cplx>& A, int n, double h) {
    double nrm = 0.0;
    for (const cplx& z : A) nrm = std::max(nrm, std::abs(z) * std::fabs(h));
    nrm *= n;
    int sq = 0;
    while (nrm > 0.25 && sq < 60) { nrm *= 0.5; ++sq; }
    const double sc = h / std::pow(2.0, sq);
    std::vector<cplx> X(A.size()), T(n * n, cplx(0)), R(n * n, cplx(0)), Tn(n * n);
    for (size_t i = 0; i < A.size(); ++i) X[i] = A[i] * sc;
    for (int i = 0; i < n; ++i) { T[i * n + i] = 1.0; R[i * n + i] = 1.0; }
    for (int k = 1; k <= 20; ++k) {
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < n; ++j) {
                cplx acc = 0.0;
                for (int l = 0; l < n; ++l) acc += T[i * n + l] * X[l * n + j];
                Tn[i * n + j] = acc / (double)k;
            }
        T = Tn;
        for (int i = 0; i < n * n; ++i) R[i] += T[i];
    }
    for (int q = 0; q < sq; ++q) {
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < n; ++j) {
                cplx acc = 0.0;
                for (int l = 0; l < n; ++l) acc += R[i * n + l] * R[l * n + j];
                Tn[i * n + j] = acc;
            }
        R = Tn;
    }
    return R;
}

// rho <- exp(h D) rho on the vectorised density matrix in `buf` (all trajectories)
static void apply_dissipator(Plan& P, c2* buf, double h, long long& launches) {
    const int npairs = (int)P.diss_gen.size();
    const int dd = P.dim * P.dim;
    for (int k = 0; k < npairs; ++k) {
        const std::vector<cplx> E = small_expm(P.diss_gen[k], dd, h);
        PairOp op{};
        for (int i = 0; i < dd * dd; ++i) op.m[i] = {E[i].real(), E[i].imag()};
        long long s_hi = 1, s_lo = 1;
        for (int i = 0; i < P.n - 1 - k; ++i) s_hi *= P.dim;            // row qudit k
        for (int i = 0; i < P.n - 1 - (k + npairs); ++i) s_lo *= P.dim;  // column qudit k + N
        const long long groups = P.D / dd;
        const long long blocks = std::min<long long>((groups + 255) / 256, (long long)P.sm_count * 16);
        dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)P.B);
        pair_op_kernel<<<grid, 256, 0, P.stream>>>(buf, P.D, P.dim, s_hi, s_lo, op);
        ++launches;
    }
    CUDA_CHECK(cudaGetLastError());
}

// mark sampling intervals that must be stepped one by one
static std::vector<char> fine_intervals(const Plan& P, int window, double rough_tol, double jump_tol,
                                        std::vector<char>& jump, std::vector<int>& dist) {
    const int nt = (int)P.times.size();
    std::vector<char> rough(nt, 0);
    jump.assign(std::max(nt - 1, 1), 0);
    auto scan = [&](auto const& pcs, const std::vector<double>& scales, auto absf) {
        for (size_t r = 0; r < pcs.size(); ++r) {
            const auto& pc = pcs[r];
            const double sc = scales[r];
            if (sc <= 0.0) continue;
            // third differences of the samples (c0 holds y_i; last sample is implied by the last piece)
            const int np = pc.pieces();
            auto y = [&](int i) { return i < np ? pc.c0[i] : pc.eval_piece(np - 1, P.times[np] - P.times[np - 1]); };
            for (int i = 1; i + 2 < nt; ++i) {
                auto d3 = y(i + 2) - 3.0 * y(i + 1) + 3.0 * y(i) - y(i - 1);
                if (absf(d3) > rough_tol * sc) { rough[i] = 1; rough[i + 1] = 1; }
            }
            // sample-to-sample jumps (pulse edges, the zero-padded last sample): the interval and its
            // neighbours (spline overshoot) are sub-stepped
            for (int i = 0; i + 1 < nt; ++i)
                if (absf(y(i + 1) - y(i)) > jump_tol * sc)
                    for (int j = std::max(0, i - 2); j <= std::min(nt - 2, i + 2); ++j) jump[j] = 1;
        }
    };
    for (int tr = 0; tr < P.B; ++tr)
        for (int q = 0; q < P.n_drives; ++q) {
            const DriveTables& T = P.tabs[tr][q];
            scan(T.coef, T.coef_scale, [](cplx z) { return std::abs(z); });
            scan(T.det, T.det_scale, [](double z) { return std::fabs(z); });
        }
    if (P.has_slm) {  // the 0 -> 1 switch of the masked interaction is a jump like a pulse edge
        std::vector<PiecewiseCubic<double>> one{P.slm_coef};
        scan(one, std::vector<double>{1.0}, [](double z) { return std::fabs(z); });
    }
    std::vector<char> fine(std::max(nt - 1, 1), 0);
    for (int r = 0; r < nt; ++r)
        if (rough[r])
            for (int i = std::max(0, r - window); i <= std::min(nt - 2, r + window - 1); ++i) fine[i] = 1;
    // distance (in intervals) from interval i to the nearest non-smooth sample
    const int BIG = 1 << 28;
    dist.assign(std::max(nt - 1, 1), BIG);
    int last = -BIG;
    for (int i = 0; i < nt - 1; ++i) { if (rough[i]) last = i; dist[i] = std::min(dist[i], i - last); }
    last = BIG;
    for (int i = nt - 2; i >= 0; --i) { if (rough[i + 1]) last = i + 1; dist[i] = std::min(dist[i], last - i); }
    return fine;
}

// defaults of refine_window and rough_tol
constexpr int kRefineWindow = 8;
constexpr double kRoughTol = 1e-4;

// the interval classification of the sampling grid, cached on the plan; jump intervals count as fine
static const Plan::FineCache& interval_classes(Plan& P, int window, double rough_tol) {
    Plan::FineCache& F = P.fine_cache;
    if (!F.valid || F.window != window || F.rtol != rough_tol) {
        F.fine = fine_intervals(P, window, rough_tol, 0.05, F.jump, F.dist);
        for (size_t i = 0; i < F.fine.size(); ++i) if (F.jump[i]) F.fine[i] = 1;
        F.window = window; F.rtol = rough_tol; F.valid = true;
    }
    return F;
}

// Magnus step [a, b] appended to the program (2 exponentials for order 4)
static void add_step(const Plan& P, Program& prog, const ExpChoice& X, double a, double b, int order, double tol) {
    const double h = b - a;
    const size_t first = prog.cheb.size();
    struct DissMark {  // symmetric splitting exp(h/2 D) U(h) exp(h/2 D) around the unitary part of the step
        const Plan& P; Program& prog; size_t first; double h;
        ~DissMark() {
            if (P.has_diss && prog.cheb.size() > first) {
                prog.pre_diss[first] = 0.5 * h;
                prog.post_diss[prog.cheb.size() - 1] = 0.5 * h;
            }
        }
    } mark{P, prog, first, h};
    if (order == 4) {
        ExpParams m1;
        const ExpParams m0 = step_generator(P, a, b, &m1);
        const size_t cnt = m0.g.size();
        ExpParams E1, E2;
        E1.g.resize(cnt); E1.th.resize(cnt); E2.g.resize(cnt); E2.th.resize(cnt);
        for (size_t x = 0; x < cnt; ++x) {
            E1.g[x] = 0.5 * m0.g[x] - 2.0 * m1.g[x]; E1.th[x] = 0.5 * m0.th[x] - 2.0 * m1.th[x];
            E2.g[x] = 0.5 * m0.g[x] + 2.0 * m1.g[x]; E2.th[x] = 0.5 * m0.th[x] + 2.0 * m1.th[x];
        }
        E1.w = 0.5 * h; E2.w = 0.5 * h;
        E1.wc = 0.5 * m0.wc - 2.0 * m1.wc; E2.wc = 0.5 * m0.wc + 2.0 * m1.wc;
        add_exponential(P, prog, E1, tol, X);
        add_exponential(P, prog, E2, tol, X);
    } else {
        add_exponential(P, prog, step_generator(P, a, b), tol, X);
    }
}

// number of sub-steps of a jump interval from the a-priori Magnus remainder bound
static int jump_substeps(const Plan& P, double a, double b, double magnus_tol) {
    ExpParams m1;
    const double rh = generator_rho(P, step_generator(P, a, b, &m1));
    double b1 = 0.0;
    for (int tr = 0; tr < P.B; ++tr) {
        double acc = 0.0;
        for (int q = 0; q < P.n_drives; ++q)
            for (int k = 0; k < P.n; ++k) acc += std::abs(m1.g[pidx(P, tr, q, k)]) + std::fabs(m1.th[pidx(P, tr, q, k)]);
        b1 = std::max(b1, acc);
    }
    const double est = 8.0 * rh * rh * rh * b1 / 60.0;  // (2 rho)^3 |B1| / 60
    int nsub = (int)std::ceil(std::pow(std::max(est / magnus_tol, 1.0), 0.25));
    return std::min(std::max(nsub, 1), 32);
}

static void ensure_aux_buffers(Plan& P) {
    for (int i = 0; i < 6; ++i)
        if (!P.aux[i]) P.aux[i].reset(P, (size_t)P.D * P.B);
}

// ---- Monte-Carlo wave-function propagation (collapse operators without a density matrix) ------------------------
static constexpr double kMcwfJumpPerStep = 0.01;   // bound on N * rate_max * step

static void propagate_mcwf(Plan& P, double t_start, double t_stop, const pb200_run_opts* o, pb200_run_stats* stats) {
    const double eps = 1e-12;
    const int nt = (int)P.times.size();
    pb200_run_stats st{};
    ExpChoice X;   // Chebyshev, no forwarding
    X.passes = plan_passes(P.n, kStageTileBits, kMaxExtraBits);
    const std::vector<char>& jump = interval_classes(P, kRefineWindow, kRoughTol).jump;
    const int K = (o && o->max_step_samples > 0) ? o->max_step_samples : 1;
    DecayTable dt{};
    for (int dgt = 0; dgt < P.dim; ++dgt) {
        double g = 0.0;
        for (const auto& l : P.jump_ldl) g += l[dgt];
        dt.gamma[dgt] = g;
    }
    const long long blocks = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 8);
    dim3 bgrid((unsigned)std::max<long long>(blocks, 1), (unsigned)P.B);
    EventPair evs;
    evs.start(P.stream);
    std::vector<double> norms(P.B), occ((size_t)P.dim * P.n);
    DevBuf<double> d_occ(P, (size_t)P.dim * P.n);   // populations [digit][qudit]
    std::uniform_real_distribution<double> uni(0.0, 1.0);
    auto norms2 = [&]() {
        const long long nb = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 4);
        dim3 grid((unsigned)std::max<long long>(nb, 1), (unsigned)P.B);
        device_sum(P, P.d_scratch.get(), P.B, norms.data(),
                   [&] { norm2_kernel<<<grid, 256, 0, P.stream>>>(P.buf[P.cur].get(), P.D, P.d_scratch.get()); });
        st.n_launches += 1;
    };
    // K_tot = sum_c L_c^+ L_c (d x d): its norm bounds the jump rate per qudit
    const int d = P.dim;
    std::vector<cplx> Ktot((size_t)d * d, cplx(0));
    double rate_max = 0.0;
    for (const auto& kf : P.jump_ldl_full)
        for (int q = 0; q < d * d; ++q) Ktot[q] += kf[q];
    for (int a = 0; a < d; ++a) {
        double row = 0.0;
        for (int c = 0; c < d; ++c) row += std::abs(Ktot[a * d + c]);
        rate_max = std::max(rate_max, row);
    }
    // the no-jump evolution exp(-tau sum_k K_tot^(k)): one elementwise kernel when every L^+L is diagonal, else the
    // d x d matrix exp(-tau K_tot) applied to each qudit in turn (general effective-noise operators)
    auto decay = [&](double tau) {
        if (P.jump_diag) {
            mcwf_decay_kernel<<<bgrid, 256, 0, P.stream>>>(P.buf[P.cur].get(), P.D, P.n, P.dim, tau, dt);
            st.n_launches += 1;
            return;
        }
        std::vector<cplx> A((size_t)d * d);
        for (int q = 0; q < d * d; ++q) A[q] = -Ktot[q];
        const std::vector<cplx> M = small_expm(A, d, tau);
        QuditOp qo{};
        for (int q = 0; q < d * d; ++q) qo.m[q] = {M[q].real(), M[q].imag()};
        const long long nb = std::min<long long>((P.D / d + 255) / 256, (long long)P.sm_count * 8);
        long long stq = 1;
        for (int k = P.n - 1; k >= 0; --k) {  // qudit k has stride d^(n-1-k)
            qudit_op_kernel<<<dim3((unsigned)std::max<long long>(nb, 1), (unsigned)P.B), 256, 0, P.stream>>>(
                P.buf[P.cur].get(), P.D, d, stq, 1.0, qo);
            stq *= d;
        }
        st.n_launches += P.n;
    };
    const double ctol = (o && o->cheb_tol > 0) ? o->cheb_tol : 1e-11;
    double t = t_start;
    while (t < t_stop - eps) {
        const int i = find_piece(P.times, t + eps);
        const double hi_i = P.times[i + 1] - P.times[i];
        double b = P.times[std::min(i + K, nt - 1)];
        if (jump[i]) {
            const int nsub = jump_substeps(P, t, std::min(P.times[i + 1], t_stop), 1e-9);
            b = std::min(P.times[i + 1], t + hi_i / nsub);
        }
        // jump times are resolved to one step and a trajectory jumps at most once per step, so the clocks of the other
        // qudits restart at the step end: keep the jump probability of the whole register per step below 1 %, which
        // holds the resulting deficit of jumps (first order in the step) near 1e-3 of the decayed population
        if (rate_max > 0.0) b = std::min(b, t + kMcwfJumpPerStep / (P.n * rate_max));
        b = std::min(b, t_stop);
        const double h = b - t;
        // exp(-i H_eff h) ~ decay(h/2) U(h) decay(h/2)
        decay(0.25 * h);
        Program prog;
        add_step(P, prog, X, t, b, 4, ctol);
        run_program(P, prog, X, st);
        CUDA_CHECK(cudaStreamSynchronize(P.stream));
        decay(0.25 * h);
        CUDA_CHECK(cudaGetLastError());
        ++st.n_steps;
        // quantum jumps
        norms2();
        for (int tr = 0; tr < P.B; ++tr) {
            if (norms[tr] > P.thresholds[tr]) continue;
            c2* psi = P.buf[P.cur].get() + (size_t)tr * P.D;
            std::vector<double> wts(P.jump_ops.size() * (size_t)P.n);
            double tot = 0.0;
            if (!P.jump_diag) {
                // <L_c^+ L_c> on qudit k = Tr(L_c^+ L_c rho_k) with the single-qudit reduced density matrix rho_k
                std::vector<double> hr((size_t)2 * d * d);
                const long long nbq = std::min<long long>((P.D / d + 255) / 256, (long long)P.sm_count * 4);
                long long stq = 1;
                for (int k = P.n - 1; k >= 0; --k) {
                    device_sum(P, P.d_scratch.get(), hr.size(), hr.data(), [&] {
                        reduced_density_kernel<<<(unsigned)std::max<long long>(nbq, 1), 256, 0, P.stream>>>(psi, P.D, d, stq,
                                                                                                           P.d_scratch.get());
                    });
                    for (size_t op = 0; op < P.jump_ops.size(); ++op) {
                        cplx tr_k = 0.0;
                        for (int a = 0; a < d; ++a)
                            for (int c = 0; c < d; ++c)
                                tr_k += P.jump_ldl_full[op][a * d + c] * cplx(hr[2 * (c * d + a)], hr[2 * (c * d + a) + 1]);
                        const double wv = std::max(tr_k.real(), 0.0);
                        wts[op * P.n + k] = wv; tot += wv;
                    }
                    stq *= d;
                }
                st.n_launches += P.n;
            }
            // populations of every digit on every qudit
            if (P.jump_diag) {
                const long long nb = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 4);
                device_sum(P, d_occ.get(), occ.size(), occ.data(), [&] {
                    for (int dgt = 0; dgt < P.dim; ++dgt)
                        occupation_kernel<false><<<(unsigned)std::max<long long>(nb, 1), 256, sizeof(double) * P.n, P.stream>>>(
                            psi, d_occ.get() + (size_t)dgt * P.n, P.D, P.D, P.n, P.dim, dgt, 0LL);
                });
            }
            // channel (op, qudit) with probability <L^+L>
            for (size_t op = 0; P.jump_diag && op < P.jump_ops.size(); ++op)
                for (int k = 0; k < P.n; ++k) {
                    double wv = 0.0;
                    for (int dgt = 0; dgt < P.dim; ++dgt) wv += P.jump_ldl[op][dgt] * occ[(size_t)dgt * P.n + k];
                    wts[op * P.n + k] = wv; tot += wv;
                }
            if (tot <= 0.0) { P.thresholds[tr] = uni(P.rng); continue; }
            double x = uni(P.rng) * tot; size_t sel = 0;
            for (; sel + 1 < wts.size(); ++sel) { x -= wts[sel]; if (x <= 0.0) break; }
            const size_t op = sel / P.n; const int k = (int)(sel % P.n);
            QuditOp qo{};
            for (int q = 0; q < P.dim * P.dim; ++q) qo.m[q] = {P.jump_ops[op][q].real(), P.jump_ops[op][q].imag()};
            long long stq = 1;
            for (int q = 0; q < P.n - 1 - k; ++q) stq *= P.dim;
            const double scale = 1.0 / std::sqrt(std::max(wts[sel], 1e-300));  // psi <- L psi / ||L psi||
            const long long nb = std::min<long long>((P.D / P.dim + 255) / 256, (long long)P.sm_count * 8);
            qudit_op_kernel<<<(unsigned)std::max<long long>(nb, 1), 256, 0, P.stream>>>(psi, P.D, P.dim, stq, scale, qo);
            CUDA_CHECK(cudaGetLastError());
            st.n_launches += 1 + P.dim;
            P.thresholds[tr] = uni(P.rng);
            P.jump_count[tr] += 1;
        }
        t = b;
    }
    // renormalise for the caller (mcsolve returns normalised states); thresholds are kept relative to norm 1
    norms2();
    for (int tr = 0; tr < P.B; ++tr) {
        if (norms[tr] <= 0.0) continue;
        const double sc = 1.0 / std::sqrt(norms[tr]);
        scale_kernel<<<(unsigned)std::max<long long>(blocks, 1), 256, 0, P.stream>>>(P.buf[P.cur].get() + (size_t)tr * P.D, P.D, sc);
        P.thresholds[tr] /= norms[tr];  // the same decay continues from the rescaled state
        P.thresholds[tr] = std::min(P.thresholds[tr], 1.0);
    }
    CUDA_CHECK(cudaGetLastError());
    st.gpu_ms = evs.stop_ms(P.stream); st.integrator = 1; st.mean_step_samples = K;
    if (stats) *stats = st;
}

static thread_local const char* g_taylor_why = "";   // why the Taylor propagator was not taken (PB200_TAYLOR_LOG)
static bool taylor_prepare(Plan& P);
static bool taylor_worthwhile(Plan& P, double gtol);
static bool taylor_geometry(const Plan& P, PassGeom& geo, bool& tiled);
static void propagate_taylor(Plan& P, double t_start, double t_stop, const pb200_run_opts* o, pb200_run_stats* stats);

// error budget of a Taylor run: the caller's tol, else 1e-8 for states and 1e-10 for density matrices (no splitting
// error to pay for: the master equation gets the same a-priori control as a pure state, at a tighter default)
static double taylor_default_tol(const Plan& P, const pb200_run_opts* o) {
    return (o && o->tol > 0.0) ? o->tol : (P.has_diss ? 1e-10 : 1e-8);
}

// Host half of the Magnus propagator (integrators 1 and 2): the options of one call [t_start, t_stop] resolved once, the
// call's exponential choice, and the step controller -- where a step ends, the step-doubling check, accept / reject.
// Every step is error-controlled.  "Fine" intervals (next to a non-smooth sample) are never merged with their
// neighbours; elsewhere up to Kc intervals form one step.  In both cases the step may be a fraction of an interval when
// the controller or the convergence-radius cap ask for it.
struct MagnusController {
    Plan& P;
    double t_stop, eps = 1e-12;
    double gtol, tol_user, rtol, rate_allowed, rho_cap;
    bool extrap, adaptive;
    int Kmax, W, order, check_every, pw_base;
    ExpChoice X;
    const Plan::FineCache* F = nullptr;
    double Kc;                   // current smooth-step length in sampling intervals (real: < 1 means sub-steps)
    int since_check = 1 << 30;   // force a check at the first smooth step
    int n_rejected = 0;          // consecutive rejections of the current step
    bool last_fine = false;
    double smooth_len = 0.0; long long smooth_steps = 0;
    pb200_run_stats st{};
    Program prog;                // steps queued for the next flush

    MagnusController(Plan& P_, double t_start, double t_stop_, const pb200_run_opts* o) : P(P_), t_stop(t_stop_) {
        gtol = (o && o->tol != 0.0) ? o->tol : (P.has_diss ? 1e-6 : 1e-8);
        // Richardson extrapolation: on by default (extrapolate = 0 or 1), -1 switches it off
        extrap = !(o && o->extrapolate < 0);
        adaptive = gtol > 0.0;
        // defaults of max_step_samples (adaptive + extrapolated / adaptive / fixed steps)
        constexpr int kMaxStepExtrap = 32, kMaxStepAdaptive = 16, kMaxStepFixed = 4;
        Kmax = (o && o->max_step_samples > 0) ? o->max_step_samples
                                              : (adaptive ? (extrap ? kMaxStepExtrap : kMaxStepAdaptive) : kMaxStepFixed);
        W = (o && o->refine_window >= 0) ? o->refine_window : kRefineWindow;
        tol_user = (o && o->cheb_tol > 0) ? o->cheb_tol : 0.0;
        rtol = (o && o->rough_tol > 0) ? o->rough_tol : kRoughTol;
        order = (o && o->magnus_order) ? o->magnus_order : 4;
        check_every = (o && o->check_every > 0) ? o->check_every : 12;
        if (order != 2 && order != 4) fail(PB200_ERR_INVALID, "magnus_order must be 2 or 4");
        // error budget per unit of time: gtol over the whole sampling-time range
        rate_allowed = adaptive ? gtol / std::max(P.times.back() - P.times.front(), 1e-30) : 0.0;
        // order of the one-step map whose error the controller / extrapolation sees: the Lindblad splitting is
        // a symmetric 2nd-order scheme whatever the order of its unitary part
        pw_base = P.has_diss ? 2 : ((order == 4) ? 4 : 2);
        F = &interval_classes(P, W, rtol);
        // exponential: Chebyshev-Clenshaw (cost ~ full spectral width) or Lanczos (cost ~ populated spectral width);
        // auto picks Lanczos when one sampling interval already spans a Chebyshev half-width near 1, i.e. for
        // strongly blockaded registers whose high-energy states are not populated
        constexpr double kKrylovRhoPerInterval = 0.9;
        constexpr double kKrylovStateBytes = 64.0 * 1048576.0;
        const int req = o ? o->integrator : 0;
        X.krylov = req == 2;
        if (req == 0) {
            const int nt = (int)P.times.size();
            const double rh1 = generator_rho(P, step_generator(P, P.times[0], P.times[std::min(1, nt - 1)]));
            // ... or when the state no longer fits L2 (fewer, fatter iterations win once HBM-bound)
            X.krylov = rh1 > kKrylovRhoPerInterval || (double)P.D * P.B * 16.0 > kKrylovStateBytes;
        }
        // spectral half-width of one step's exponential: Chebyshev / Lanczos
        constexpr double kRhoCapChebyshev = 3.6, kRhoCapKrylov = 12.0;
        rho_cap = X.krylov ? kRhoCapKrylov : kRhoCapChebyshev;
        X.passes = plan_passes(P.n, kStageTileBits, kMaxExtraBits);
        X.dual_ok = dual_chain_ok(P, X.passes) && !P.has_diss && !X.krylov;
        X.fwd = !X.krylov && !P.has_diss && fwd_eligible(P, X.passes);
        if (X.fwd) plan_fwd_passes(P, X.fwd_passes);
        Kc = adaptive ? std::min(extrap ? 8.0 : 4.0, (double)Kmax) : (double)Kmax;
        // a call that continues where the previous one stopped (same options) inherits its step length: with "Full"
        // evaluation times every sampling interval is its own call, and re-growing the step from scratch (and paying
        // the 3x-cost check) on each of them would dominate the run
        if (adaptive && P.ctrl_Kc > 0.0 && P.ctrl_opts == options() && std::fabs(P.ctrl_t_end - t_start) < 1e-9) {
            Kc = std::min(P.ctrl_Kc, (double)Kmax);
            since_check = check_every / 2;
        }
    }

    Plan::CtrlOptions options() const { return {gtol, extrap, order, Kmax}; }

    // Chebyshev truncation per exponential: a fifth of the step's share of the error budget
    // (a hundredth inside a step-doubling check so that the estimate is not truncation noise)
    double cheb_tol_for(double h, bool check) const {
        if (tol_user > 0.0) return tol_user;
        if (!adaptive) return 1e-12;
        const double share = rate_allowed * h;
        return std::min(1e-12, std::max(2e-15, (check ? 0.01 : 0.2) * share));
    }

    void flush() {
        if (prog.cheb.empty()) return;
        run_program(P, prog, X, st);
        CUDA_CHECK(cudaStreamSynchronize(P.stream));  // tables are copied asynchronously from prog
        prog = Program();
    }

    void copy_state(const DevBuf<c2>& dst, const DevBuf<c2>& src) {
        CUDA_CHECK(cudaMemcpyAsync(dst.get(), src.get(), sizeof(c2) * P.D * P.B, cudaMemcpyDeviceToDevice, P.stream));
    }

    double max_diff2(const DevBuf<c2>& x, const DevBuf<c2>& y) {
        const int nb = std::min(P.B, 4096);
        const long long blocks = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 4);
        dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)nb);
        std::vector<double> d2(nb);
        device_sum(P, P.d_scratch.get(), nb, d2.data(),
                   [&] { diffnorm2_kernel<<<grid, 256, 0, P.stream>>>(x.get(), y.get(), P.D, P.d_scratch.get()); });
        st.n_launches += 1;
        double e = 0.0;
        for (double v : d2) e = std::max(e, v);
        return e;
    }

    // end of the step from t, which lies in sampling interval i
    double step_end(double t, int i) {
        const int nt = (int)P.times.size();
        const double hi_i = P.times[i + 1] - P.times[i];
        const bool is_fine = F->fine[i] != 0;
        if (is_fine != last_fine) { since_check = 1 << 30; last_fine = is_fine; }  // re-validate on region change
        double Kuse = is_fine ? std::min(Kc, 1.0) : Kc;
        {   // keep the step inside the convergence radius of the Magnus expansion: the spectral
            // half-width of int H dt over the step stays below rho_cap (~pi)
            const double b1 = std::min(P.times[i + 1], t_stop);
            const double frac = (b1 - t) / hi_i;  // fraction of a sampling interval covered by this probe
            const double rho_per_sample = generator_rho(P, step_generator(P, t, b1)) / std::max(frac, 1e-9);
            Kuse = std::min(Kuse, rho_cap / std::max(rho_per_sample, 1e-12));
        }
        double b;
        if (Kuse >= 1.0) {
            int K = std::max(1, std::min((int)std::floor(Kuse + 1e-9), Kmax));
            if (is_fine) {
                b = P.times[i + 1];
            } else {
                // graded steps: no longer than half the distance to the nearest non-smooth sample on either side
                K = std::max(1, std::min(K, F->dist[i] / 2));
                int j = i, cnt = 0;
                while (j < nt - 1 && !F->fine[j] && cnt < K && (cnt == 0 || 2 * (cnt + 1) <= std::max(F->dist[j], 2))) { ++j; ++cnt; }
                b = P.times[j];
            }
        } else {
            const int nsub = std::min(64, (int)std::ceil(1.0 / std::max(Kuse, 1.0 / 64.0) - 1e-9));
            b = std::min(P.times[i + 1], t + hi_i / nsub);
        }
        if (F->jump[i] && order == 4) {  // a-priori sub-stepping of sample-to-sample jumps
            constexpr double kMagnusTol = 1e-11;
            const int nsub = jump_substeps(P, t, std::min(P.times[i + 1], t_stop), kMagnusTol);
            if (nsub > 1) b = std::min(b, t + hi_i / nsub);
        }
        b = std::min(b, t_stop);
        if (b <= t + eps) b = std::min(P.times[std::min(i + 1, nt - 1)], t_stop);
        return b;
    }

    // step doubling: one `step` of h from the current state (saved in aux[save]) into aux[save + 1], then two of h/2
    // from the same state into the current state
    template <typename Step>
    void step_doubled(double a, double b, int save, const Step& step) {
        flush();
        ensure_aux_buffers(P);
        copy_state(P.aux[save], P.buf[P.cur]);
        step(a, b);
        flush();
        copy_state(P.aux[save + 1], P.buf[P.cur]);
        copy_state(P.buf[P.cur], P.aux[save]);
        const double mid = 0.5 * (a + b);
        step(a, mid);
        step(mid, b);
        flush();
    }

    // step-length update from the check of [t, b] (e: its squared distance, ctol: its Chebyshev tolerance).  Returns
    // false when the step is rejected, with the state the check saved in aux[save] restored
    bool accept(double t, double b, double h_samples, double ctol, double e, int save) {
        const int pw = extrap ? pw_base + 2 : pw_base;
        const double scale = std::pow(2.0, pw) - 1.0;
        const double err_big = std::sqrt(e) * std::pow(2.0, pw) / scale;
        st.err_estimate += std::sqrt(e) / scale;
        ++st.n_checks;
        const double rate = err_big / std::max(b - t, 1e-30);
        double factor = 2.0;
        // differences at the level of truncation / rounding noise carry no information
        const double noise = 50.0 * ctol + 1e-14;
        if (err_big > noise) factor = std::pow(0.5 * rate_allowed / rate, 1.0 / pw);
        factor = std::min(2.0, std::max(0.2, factor));
        const bool controller_limited = h_samples >= 0.9 * Kc;  // not shortened by a cap / grading
        Kc = std::min((double)Kmax, std::max(1.0 / 16.0, h_samples * factor));
        // re-check soon after a big cut, and while a controller-limited step is still growing at the
        // maximum rate (so that the step recovers quickly after a non-smooth stretch)
        since_check = (factor < 0.7) ? check_every - 2 : ((factor >= 1.9 && controller_limited) ? check_every - 3 : 0);
        // the state kept by a check is the pair of half steps, whose own error is err_big / 2^pw; if even
        // that exceeds the step's share of the budget the step is REJECTED: restore the saved state and
        // retry with the shortened step (at most 4 times in a row, then accept and let the budget absorb it)
        const double kept_rate = std::sqrt(e) / scale / std::max(b - t, 1e-30);
        if (kept_rate > rate_allowed && n_rejected < 4 && h_samples > 1.0 / 16.0 + 1e-12) {
            copy_state(P.buf[P.cur], P.aux[save]);
            st.err_estimate -= std::sqrt(e) / scale;
            ++n_rejected; ++st.n_rejected;
            since_check = 1 << 30;
            return false;
        }
        n_rejected = 0;
        return true;
    }

    // Richardson-extrapolated step: one CF4 step of h and two of h/2 from the same state,
    // psi <- R2 + (R2 - R1) / (2^p - 1); the symmetric scheme gains two orders (6th for CF4).  Uses aux[0..3]
    void extrap_step(double a, double b, double ctol) {
        flush();
        ensure_aux_buffers(P);
        const double sc = std::pow(2.0, pw_base) - 1.0;
        const long long total = P.D * (long long)P.B;
        const long long nb = std::min<long long>((total + 255) / 256, (long long)P.sm_count * 16);
        if (X.dual_ok) {
            // the h branch and the h/2 branch start from the same state and are independent: they run as two
            // chains sharing every kernel launch, each in its own buffers (no state copies at all)
            const double mid = 0.5 * (a + b);
            Program big, half;
            add_step(P, big, X, a, b, order, ctol);
            add_step(P, half, X, a, mid, order, ctol);
            add_step(P, half, X, mid, b, order, ctol);
            c2* Y = P.buf[P.cur].get();
            c2* others[6]; int k = 0;
            for (int i = 0; i < 3; ++i) if (i != P.cur) others[k++] = P.buf[i].get();
            for (int i = 0; i < 4; ++i) others[k++] = P.aux[i].get();
            Chain ch[2];
            ch[0].prog = &half; ch[0].psi = Y; for (int i = 0; i < 3; ++i) ch[0].pool[i] = others[i];
            ch[1].prog = &big;  ch[1].psi = Y; for (int i = 0; i < 3; ++i) ch[1].pool[i] = others[3 + i];
            run_chains(P, ch, 2, X, st);
            c2* res = ch[0].result();
            axpby_kernel<<<(unsigned)nb, 256, 0, P.stream>>>(res, ch[1].result(), 1.0 + 1.0 / sc, -1.0 / sc, total);
            CUDA_CHECK(cudaGetLastError());
            st.n_launches += 1;
            // make `res` the current state buffer (swap handles if it lives in the aux set)
            bool found = false;
            for (int i = 0; i < 3; ++i) if (P.buf[i].get() == res) { P.cur = i; found = true; }
            if (!found)
                for (int i = 0; i < 4; ++i) if (P.aux[i].get() == res) { std::swap(P.aux[i], P.buf[P.cur]); break; }
            if (!one_uniform_state(P))
                CUDA_CHECK(cudaStreamSynchronize(P.stream));  // tables of big/half were uploaded from this scope
            return;
        }
        step_doubled(a, b, 0, [&](double x, double y) { add_step(P, prog, X, x, y, order, ctol); });
        axpby_kernel<<<(unsigned)nb, 256, 0, P.stream>>>(P.buf[P.cur].get(), P.aux[1].get(), 1.0 + 1.0 / sc, -1.0 / sc, total);
        CUDA_CHECK(cudaGetLastError());
        st.n_launches += 1;
    }

    void run(double t) {
        const size_t flush_doubles = (size_t)8 << 20;  // 64 MiB of tables per chunk
        const bool can_aux = (P.D * (long long)P.B) <= (1LL << 31);
        while (t < t_stop - eps) {
            const int i = find_piece(P.times, t + eps);
            const double b = step_end(t, i);
            const double h_samples = (b - t) / (P.times[i + 1] - P.times[i]);
            if (adaptive && since_check >= check_every && can_aux) {
                // check: the step doubled, keeping the pair of half steps (the extrapolated step itself uses aux[0..3])
                const double ctol = cheb_tol_for(b - t, true);
                const int save = extrap ? 4 : 0;
                if (extrap) step_doubled(t, b, save, [&](double x, double y) { extrap_step(x, y, ctol); });
                else step_doubled(t, b, save, [&](double x, double y) { add_step(P, prog, X, x, y, order, ctol); });
                if (!accept(t, b, h_samples, ctol, max_diff2(P.buf[P.cur], P.aux[save + 1]), save)) continue;
            } else if (extrap && can_aux) {
                extrap_step(t, b, adaptive ? cheb_tol_for(b - t, false) : 1e-13);
                ++since_check;
            } else {
                add_step(P, prog, X, t, b, order, cheb_tol_for(b - t, false));
                ++since_check;
                if (prog.tables.size() > flush_doubles) flush();
            }
            ++st.n_steps; smooth_len += h_samples; ++smooth_steps;
            t = b;
        }
        flush();
        P.ctrl_Kc = Kc; P.ctrl_opts = options(); P.ctrl_t_end = t_stop;
    }
};

static void propagate_magnus(Plan& P, double t_start, double t_stop, const pb200_run_opts* o, pb200_run_stats* stats) {
    MagnusController M(P, t_start, t_stop, o);
    EventPair evs;
    evs.start(P.stream);
    M.run(t_start);
    M.st.gpu_ms = evs.stop_ms(P.stream);
    M.st.mean_step_samples = M.smooth_steps ? M.smooth_len / M.smooth_steps : 0.0;
    M.st.integrator = M.X.krylov ? 2 : 1;
    if (stats) *stats = M.st;
}

static void propagate(Plan& P, double t_start, double t_stop, const pb200_run_opts* o, pb200_run_stats* stats) {
    if (!P.state_set) fail(PB200_ERR_STATE, "pb200_propagate: no state set (call pb200_state_set first)");
    check_drives_set(P, "pb200_propagate");
    const double tlo = P.times.front(), thi = P.times.back();
    const double eps = 1e-12;
    if (t_start < tlo - eps || t_stop > thi + eps || t_stop < t_start)
        fail(PB200_ERR_INVALID, "pb200_propagate: [%g, %g] outside sampling times [%g, %g]", t_start, t_stop, tlo, thi);
    t_start = std::max(t_start, tlo); t_stop = std::min(t_stop, thi);
    if (P.has_collapse) { propagate_mcwf(P, t_start, t_stop, o, stats); return; }
    {   // integrator 3 / auto: the time-dependent Taylor propagator wherever it applies (global drive of any phase,
        // d = 2, one state) unless the caller steers the Magnus controller explicitly
        const int req = o ? o->integrator : 0;
        if (req < 0 || req > 3) fail(PB200_ERR_INVALID, "integrator must be 0 (auto), 1, 2 or 3");
        bool want = req == 3;
        if (req == 0) {
            const bool steered = o && (o->max_step_samples > 0 || o->tol < 0.0 || o->extrapolate < 0 || o->check_every > 0 ||
                                       o->cheb_tol > 0.0 || (o->magnus_order != 0 && o->magnus_order != 4));
            want = !steered && t_stop > t_start;   // short calls too ("Full" evaluation times: one call per sampling
                                                   // interval = one exact cubic step of ~10 orders, against ~50
                                                   // H-applies for a Richardson-CF4 step of the same length)
        }
        if (want) {
            PassGeom geo;
            bool tiled = false;
            const bool ok = taylor_prepare(P) && taylor_geometry(P, geo, tiled) &&
                            (req == 3 || taylor_worthwhile(P, taylor_default_tol(P, o)));
            if (ok) { propagate_taylor(P, t_start, t_stop, o, stats); return; }
            if (env_int("PB200_TAYLOR_LOG", 0)) fprintf(stderr, "taylor not taken: %s\n", g_taylor_why);
            if (req == 3)
                fail(PB200_ERR_UNSUPPORTED, "integrator 3 (Taylor) needs a d = 2 register whose drive rows are multiples of one row "
                                            "(per-qubit static factors / detuning offsets allowed), no collapse operators / SLM mask, "
                                            "and a dissipator of one generator without single-bit flips: %s",
                     g_taylor_why);
        }
    }
    propagate_magnus(P, t_start, t_stop, o, stats);
}

// ---- time-dependent Taylor propagator (one drive time shape, its phase constant or moving, d = 2) -----------------
// Replaces the whole Magnus / exponential machinery above where it applies (C2, C5; C4 batches through per-qubit static
// factors, taylor_separable): the interpolated coefficients
// are polynomials in u = (t-a)/h on a step, the solution is the Taylor series in u (kernels.cuh,
// stage_d2_taylor_kernel), one H-apply per order.  A step spans rho = h W ~ 10 (W = spectral half-width) instead of
// the ~1.5 a Richardson-CF4 exponential manages, and pays no Chebyshev start-up per exponential: ~1 H-apply per ns on
// C2 against 6.9.  Error = fit residual of the splines (measured) + Taylor remainder (majorant bound) -- both a priori,
// so a run never synchronises with the host.

// Separable structure of a batch of drive tables, read off the samples (the interpolants are linear in the samples and
// share their knots):  coef_{b,k}[i] = a_{b,k} * coef_ref[i]  and  det_{b,k}[i] = det_{0,0}[i] + sum_s c_{b,k,s} m_s[i]
// with ONE reference drive row (the largest one) and at most max_shapes common shapes m_s (max |m_s| = 1): detuning
// maps, masks and doppler noise each add one.  Greedy: the difference row with the largest residual becomes the next
// shape, normalised at that sample, and every row is fitted again on all shapes.  cs(b,k,i) / ds(b,k,i) return the
// samples.  Least-squares factors with extended-precision sums (4001 same-sign terms: a plain double sum is only good
// to ~1e-13, which is the size of the residual being tested).  Host only; also reachable through
// pb200_host_taylor_separable (one shape) and pb200_host_taylor_shapes.
static const char* const kWhyDriveRows = "a drive row is not a constant multiple of the reference row";
struct SeparableFit {
    bool ok = false;
    const char* why = "";
    int ref_b = 0, ref_k = 0;       // reference drive row
    cplx big = 0.0; double scale = 0.0;
    std::vector<cplx> a;            // [B][N]
    int ns = 0;                     // shapes
    std::vector<double> c;          // [B][N][ns]
    std::vector<std::vector<double>> m;   // [ns][nt]
};

// least-squares factors of every difference row on the shapes F.m (normal equations in extended precision; the greedy
// shapes are residuals of the earlier fit, so the system is close to diagonal); max |residual| and where it is
template <class DS>
static double taylor_shape_factors(int B, int N, int nt, DS ds, SeparableFit& F, int& rb, int& rk, int& ri) {
    typedef long double ld;
    const int S = F.ns;
    std::vector<ld> G((size_t)S * S, 0.0L);
    for (int s = 0; s < S; ++s)
        for (int u = 0; u < S; ++u)
            for (int i = 0; i < nt; ++i) G[(size_t)s * S + u] += (ld)F.m[s][i] * F.m[u][i];
    F.c.assign((size_t)B * N * S, 0.0);
    double emax = -1.0;
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < N; ++k) {
            std::vector<ld> A(G), x(S, 0.0L);
            for (int s = 0; s < S; ++s)
                for (int i = 0; i < nt; ++i) x[s] += (ld)(ds(b, k, i) - ds(0, 0, i)) * F.m[s][i];
            for (int s = 0; s < S; ++s)   // Gaussian elimination (symmetric positive definite: no pivoting)
                for (int u = s + 1; u < S; ++u) {
                    const ld f = A[(size_t)u * S + s] / A[(size_t)s * S + s];
                    for (int w = s; w < S; ++w) A[(size_t)u * S + w] -= f * A[(size_t)s * S + w];
                    x[u] -= f * x[s];
                }
            for (int s = S - 1; s >= 0; --s) {
                for (int w = s + 1; w < S; ++w) x[s] -= A[(size_t)s * S + w] * x[w];
                x[s] /= A[(size_t)s * S + s];
            }
            double* cc = F.c.data() + ((size_t)b * N + k) * S;
            for (int s = 0; s < S; ++s) cc[s] = (double)x[s];
            for (int i = 0; i < nt; ++i) {
                double r = ds(b, k, i) - ds(0, 0, i);
                for (int s = 0; s < S; ++s) r -= cc[s] * F.m[s][i];
                if (std::fabs(r) > emax) { emax = std::fabs(r); rb = b; rk = k; ri = i; }
            }
        }
    return emax;
}

template <class CS, class DS>
static SeparableFit taylor_separable(int B, int N, int nt, CS cs, DS ds, int max_shapes = 1) {
    SeparableFit F;
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < N; ++k)
            for (int i = 0; i < nt; ++i) {
                const cplx y = cs(b, k, i);
                if (std::abs(y) > F.scale) { F.scale = std::abs(y); F.big = y; F.ref_b = b; F.ref_k = k; }
            }
    const double scale = F.scale;
    F.a.assign((size_t)B * N, cplx(1.0, 0.0));
    long double ref2 = 0.0L;
    for (int i = 0; i < nt; ++i) ref2 += (long double)std::norm(cs(F.ref_b, F.ref_k, i));
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < N; ++k) {
            cplx aa = 0.0;
            if (ref2 > 0.0L) {
                long double sr = 0.0L, si = 0.0L;
                for (int i = 0; i < nt; ++i) {
                    const cplx z = cs(b, k, i) * std::conj(cs(F.ref_b, F.ref_k, i));
                    sr += (long double)z.real(); si += (long double)z.imag();
                }
                aa = cplx((double)(sr / ref2), (double)(si / ref2));
            }
            for (int i = 0; i < nt; ++i)
                if (std::abs(cs(b, k, i) - aa * cs(F.ref_b, F.ref_k, i)) > 2e-13 * std::max(scale, 1e-300)) {
                    F.why = kWhyDriveRows;
                    return F;
                }
            F.a[(size_t)b * N + k] = (ref2 > 0.0L) ? aa : cplx(0.0, 0.0);
        }
    // every detuning row = the reference row (trajectory 0, qubit 0) + sum_s c_s x common shape m_s
    double dscale = 0.0;
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < N; ++k)
            for (int i = 0; i < nt; ++i) dscale = std::max(dscale, std::fabs(ds(b, k, i)));
    int mb = -1, mk = -1, mi = 0; double emax = 0.0;
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < N; ++k)
            for (int i = 0; i < nt; ++i) {
                const double e = std::fabs(ds(b, k, i) - ds(0, 0, i));
                if (e > emax) { emax = e; mb = b; mk = k; mi = i; }
            }
    F.c.clear();
    F.m.clear();
    if (emax > 1e-13 * std::max(dscale, 1e-300)) {
        for (;;) {
            if (F.ns == max_shapes) {
                F.why = max_shapes == 1 ? "a detuning row is not the reference row plus a multiple of the common shape"
                                        : "the detuning rows need more than 4 time shapes (detuning maps, masks, noise)";
                return F;
            }
            // the residual row (mb, mk) of the fit so far, normalised at its largest sample, is the next shape
            std::vector<double> row(nt);
            for (int i = 0; i < nt; ++i) {
                double r = ds(mb, mk, i) - ds(0, 0, i);
                for (int s = 0; s < F.ns; ++s) r -= F.c[((size_t)mb * N + mk) * F.ns + s] * F.m[s][i];
                row[i] = r;
            }
            const double norm = row[mi];
            for (int i = 0; i < nt; ++i) row[i] /= norm;
            F.m.push_back(std::move(row));
            ++F.ns;
            if (taylor_shape_factors(B, N, nt, ds, F, mb, mk, mi) <= 2e-13 * std::max(dscale, 1e-300)) break;
        }
    }
    F.ok = true;
    return F;
}

// per-trajectory device table image (a unit per BIT position, c per (shape,) bit position) with drive unit `unit`
static std::vector<double> taylor_table(const Plan& P, cplx unit) {
    const Plan::TaylorCache& C = P.tay;
    const int N = P.n, B = P.B;
    const int stride = C.tab_shapes ? taylor_table_stride(N, C.tab_shapes) : d2_table_stride(N);
    std::vector<double> tab((size_t)B * stride, 0.0);
    for (int b = 0; b < B; ++b) {
        double* t = tab.data() + (size_t)b * stride;
        for (int k = 0; k < N; ++k) {
            const int p = N - 1 - k;
            const cplx au = C.a[(size_t)b * N + k] * unit;
            const cplx g = (C.conj_cols && k >= N / 2) ? -std::conj(au) : au;   // column qudit k of vec(rho)
            t[2 * p] = g.real(); t[2 * p + 1] = g.imag();
            for (int s = 0; s < C.ns; ++s) t[2 * N + s * N + p] = C.c[((size_t)b * N + k) * C.ns + s];
        }
    }
    return tab;
}

// Can the Taylor stage apply this dissipator (TaylorArgs::dw, df)?  d = 2, the same generator on every atom, and no entry
// that flips exactly one bit of an atom's (row, column) pair: Gen = diagonal + "both bits flip" entries.  Pulser's
// dephasing, relaxation and depolarizing channels qualify, as does any set of collapse operators each of which is
// diagonal or off-diagonal; an operator that mixes the two does not.
static Plan::DissTaylor diss_taylor_analyse(const std::vector<std::vector<cplx>>& gen, int dim) {
    Plan::DissTaylor T;
    if (dim != 2) { T.why = "a master equation of d = 3 levels: the Taylor propagator takes d = 2 only"; return T; }
    const std::vector<cplx>& G = gen[0];
    double scale = 0.0;
    for (const std::vector<cplx>& g : gen)
        for (const cplx& z : g) scale = std::max(scale, std::abs(z));
    const double tiny = 1e-15 * scale;
    for (const std::vector<cplx>& g : gen)
        for (int i = 0; i < 16; ++i)
            if (std::abs(g[i] - G[i]) > tiny) { T.why = "the atoms carry different dissipator generators"; return T; }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j)
            if (((i ^ j) == 1 || (i ^ j) == 2) && std::abs(G[i * 4 + j]) > tiny) {
                T.why = "the dissipator has single-bit-flip entries (a collapse operator mixes diagonal and off-diagonal "
                        "elements; each one diagonal or each one off-diagonal qualifies)";
                return T;
            }
    auto c = [](cplx z) { return c2{z.real(), z.imag()}; };
    const cplx g0 = G[0], g1 = G[5], g2 = G[10], g3 = G[15];   // pair value i = 2 row bit + column bit
    T.dw[0] = c(g0 * (double)gen.size()); T.dw[1] = c(g2 - g0); T.dw[2] = c(g1 - g0); T.dw[3] = c(g0 - g1 - g2 + g3);
    double row = 0.0, col = 0.0;
    for (int i = 0; i < 4; ++i) {
        T.df[i] = c(G[i * 4 + (3 - i)]);
        T.flip = T.flip || G[i * 4 + (3 - i)] != 0.0;
        row = std::max(row, std::abs(G[i * 5]) + std::abs(G[i * 4 + (3 - i)]));
        col = std::max(col, std::abs(G[i * 5]) + std::abs(G[(3 - i) * 4 + i]));
    }
    // ||Gen||_2 <= sqrt(||Gen||_1 ||Gen||_inf), one per atom
    T.norm = (double)gen.size() * std::max(row, col);
    T.ok = true;
    return T;
}

static const char* const kWhyMovingPhaseRho =
    "the drive phase moves and the drive rows are not multiples of one row: on a density matrix a moving phase needs "
    "one global drive shape (per-qubit static factors allowed), whose columns drive -conj(omega(t))";
static const char* const kWhyMovingPhaseShards =
    "the drive phase moves: vec(rho) shards take a drive of one phase (a moving phase runs on whole density matrices)";

// the drive relative to the phase of its largest sample (real and imaginary parts), per-(trajectory, qubit) static
// factors, device table
static bool taylor_prepare(Plan& P) {
    Plan::TaylorCache& C = P.tay;
    g_taylor_why = "structure (d, drives, collapse / mask, interpolation order)";
    if (P.has_diss && !P.diss_tay.ok) { g_taylor_why = P.diss_tay.why; return false; }
    if (!is_d2path(P)) return false;
    if (P.has_collapse || P.has_slm) return false;
    if (P.desc.interp_order != 3 && P.desc.interp_order != 1) return false;
    if (C.valid) { g_taylor_why = C.ok ? "" : C.why; return C.ok; }
    C.valid = true; C.ok = false;
    const int N = P.n, B = P.B, nt = (int)P.times.size();
    auto rows_of = [&](int b) { return (int)P.tabs[b][0].coef.size(); };
    auto coef_pc = [&](int b, int k) -> const PiecewiseCubic<cplx>& { return P.tabs[b][0].coef[rows_of(b) == 1 ? 0 : k]; };
    auto det_pc = [&](int b, int k) -> const PiecewiseCubic<double>& { return P.tabs[b][0].det[rows_of(b) == 1 ? 0 : k]; };
    // row pointers once: the fit reads every sample of every row several times
    std::vector<const PiecewiseCubic<cplx>*> crow((size_t)B * N);
    std::vector<const PiecewiseCubic<double>*> drow((size_t)B * N);
    for (int b = 0; b < B; ++b)
        for (int k = 0; k < N; ++k) { crow[(size_t)b * N + k] = &coef_pc(b, k); drow[(size_t)b * N + k] = &det_pc(b, k); }
    const int npc = nt - 1;   // pieces of every interpolant; sample i = c0[i], the last one = y_last
    auto cs = [&](int b, int k, int i) { const PiecewiseCubic<cplx>* pc = crow[(size_t)b * N + k]; return i < npc ? pc->c0[i] : pc->y_last; };
    auto ds = [&](int b, int k, int i) { const PiecewiseCubic<double>* pc = drow[(size_t)b * N + k]; return i < npc ? pc->c0[i] : pc->y_last; };
    SeparableFit F = taylor_separable(B, N, nt, cs, ds, PB200_TAYLOR_SMAX);
    // vec(rho) (lindblad.doubled_spec): column qudit k + N/2 drives -conj(row k).  Under a moving phase that is no
    // multiple of the row's drive, so the drive is fitted on the row half (each column qudit reads its row's samples, and
    // gets the row's factor a) and the table conjugates on the column bits (TaylorCache::conj_cols).  The detuning rows
    // are fitted whole, as with a constant phase
    const int n2 = N / 2;
    auto doubled_fit = [&](SeparableFit& out) {
        double scale = 0.0;
        for (int b = 0; b < B; ++b)
            for (int k = 0; k < N; ++k)
                for (int i = 0; i < nt; ++i) scale = std::max(scale, std::abs(cs(b, k, i)));
        for (int b = 0; b < B; ++b)
            for (int k = 0; k < n2; ++k)
                for (int i = 0; i < nt; ++i)
                    if (std::abs(cs(b, k + n2, i) + std::conj(cs(b, k, i))) > 2e-13 * std::max(scale, 1e-300)) {
                        out.why = kWhyMovingPhaseRho;
                        return false;
                    }
        out = taylor_separable(B, N, nt, [&](int b, int k, int i) { return cs(b, k < n2 ? k : k - n2, i); }, ds,
                               PB200_TAYLOR_SMAX);
        if (out.why == kWhyDriveRows) out.why = kWhyMovingPhaseRho;
        return out.ok;
    };
    bool conj_cols = false;
    if (!F.ok && P.has_diss && F.why == kWhyDriveRows) {
        SeparableFit Fd;
        if (!doubled_fit(Fd)) { g_taylor_why = C.why = Fd.why; return false; }
        F = Fd;
        conj_cols = true;
    }
    if (!F.ok) {
        g_taylor_why = C.why = F.why;
        return false;
    }
    const double scale = F.scale;
    const cplx unit = scale > 0.0 ? F.big / scale : cplx(1.0, 0.0);
    const cplx cu = std::conj(unit);
    const PiecewiseCubic<cplx>& ref = coef_pc(F.ref_b, F.ref_k);
    const int np = ref.pieces();
    C.om = PiecewiseCubic<double>();
    C.om.c0.resize(np); C.om.c1.resize(np); C.om.c2.resize(np); C.om.c3.resize(np);
    C.om_im = C.om;
    C.phase_moves = false;
    for (int i = 0; i < np; ++i) {
        const double hi = P.times[i + 1] - P.times[i];
        const cplx v0 = ref.c0[i] * cu, v1 = ref.c1[i] * cu, v2 = ref.c2[i] * cu, v3 = ref.c3[i] * cu;
        const double im = std::max(std::max(std::fabs(v0.imag()), std::fabs(v1.imag()) * hi),
                                   std::max(std::fabs(v2.imag()) * hi * hi, std::fabs(v3.imag()) * hi * hi * hi));
        if (im > 1e-13 * scale) C.phase_moves = true;
        C.om.c0[i] = v0.real(); C.om.c1[i] = v1.real(); C.om.c2[i] = v2.real(); C.om.c3[i] = v3.real();
        C.om_im.c0[i] = v0.imag(); C.om_im.c1[i] = v1.imag(); C.om_im.c2[i] = v2.imag(); C.om_im.c3[i] = v3.imag();
    }
    C.om.y_last = (ref.y_last * cu).real();
    C.om_im.y_last = (ref.y_last * cu).imag();
    if (!C.phase_moves) C.om_im = PiecewiseCubic<double>();   // constant phase: the real drive of before, exactly
    if (P.has_diss && C.phase_moves) {
        if (P.shard_bits) { g_taylor_why = C.why = kWhyMovingPhaseShards; return false; }
        // a phase that moves within the whole fit's tolerance: the row-half fit all the same (the reference row, and with
        // it unit and omega, is the same one: a column sample is never larger than its row's)
        if (!conj_cols) {
            SeparableFit Fd;
            if (!doubled_fit(Fd) || Fd.ref_b != F.ref_b || Fd.ref_k != F.ref_k || Fd.big != F.big) {
                g_taylor_why = C.why = kWhyMovingPhaseRho;
                return false;
            }
            F = Fd;
            conj_cols = true;
        }
    }
    C.conj_cols = conj_cols;
    C.unit = {unit.real(), unit.imag()};
    C.a = F.a; C.c = F.c; C.ns = F.ns;
    for (int s = 0; s < C.ns; ++s) C.shape[s] = make_interpolant<double>(P.times.data(), F.m[s].data(), nt, P.desc.interp_order);
    C.drive_uniform = B == 1 && !P.has_diss;   // vec(rho) always runs the batch gather (stage kernels with DISS)
    C.a_sum_max = 0.0;
    for (int s = 0; s < PB200_TAYLOR_SMAX; ++s) C.c_sum_max[s] = 0.0;
    for (int b = 0; b < B; ++b) {
        double sa = 0.0, sc[PB200_TAYLOR_SMAX] = {};
        for (int k = 0; k < N; ++k) {
            sa += std::abs(C.a[(size_t)b * N + k]);
            for (int s = 0; s < C.ns; ++s) sc[s] += std::fabs(C.c[((size_t)b * N + k) * C.ns + s]);
            if (std::abs(C.a[(size_t)b * N + k] - cplx(1.0, 0.0)) > 0.0) C.drive_uniform = false;
        }
        C.a_sum_max = std::max(C.a_sum_max, sa);
        for (int s = 0; s < C.ns; ++s) C.c_sum_max[s] = std::max(C.c_sum_max[s], sc[s]);
    }
    C.uniform = C.drive_uniform && C.ns == 0;
    // a uniform drive keeps its gather with local detuning (stage_d2_taylor_kernel<true, ..., PB200_TAYLOR_SMAX>)
    C.tab_shapes = (C.ns > 1 || (C.drive_uniform && C.ns == 1)) ? PB200_TAYLOR_SMAX : 0;
    if (!C.uniform) {   // static device table: a unit per BIT position (re, im), c per (shape,) bit position
        C.tab_host = taylor_table(P, unit);
        C.d_tab.reset(P, C.tab_host.size());
        CUDA_CHECK(cudaMemcpyAsync(C.d_tab.get(), C.tab_host.data(), C.tab_host.size() * sizeof(double), cudaMemcpyHostToDevice,
                                   P.stream));
        C.tab_unit = C.unit;
    }
    C.w_knot.clear();
    C.ok = true;
    return true;
}

// Before a step whose drive unit differs from the one the device table holds (a step of one phase other than the
// reference's, TaylorStep::drive == 1): upload the table with that unit.  The host image goes into `keep`, which the
// caller holds until its stream has run the copy.
static void taylor_table_unit(Plan& P, c2 unit, std::deque<std::vector<double>>& keep) {
    Plan::TaylorCache& C = P.tay;
    if (C.uniform || (unit.x == C.tab_unit.x && unit.y == C.tab_unit.y)) return;
    keep.push_back(taylor_table(P, cplx(unit.x, unit.y)));
    CUDA_CHECK(cudaMemcpyAsync(C.d_tab.get(), keep.back().data(), keep.back().size() * sizeof(double), cudaMemcpyHostToDevice,
                               P.stream));
    C.tab_unit = unit;
}

// centre and half-width of  Dint - th n_from - sum_s mv_s sum_k c_{k,s} n_k + om X  over the batch: the rigorous bounds
// build_tables gives the Chebyshev path (per-excitation-number bounds of the shared Dint where they exist), without its
// tables.  With local detuning e_k = sum_s mv_s c_{k,s} on a uniform drive, the local term of the excitation-count-c
// states lies between minus the sums of the c largest and of the c smallest e_k.
static void taylor_bounds(const Plan& P, double om, double th, const double* mv, double& centre, double& half) {
    const int N = P.n;
    const Plan::TaylorCache& C = P.tay;
    double lo = 1e300, hi = -1e300;
    const bool caseA = C.drive_uniform && P.has_interaction && P.dint_shared &&
                       P.desc.drives[0].state_from == P.desc.rydberg_state && !P.dmin_cnt.empty();
    if (caseA) {
        const double dr = std::fabs(om) * N;
        std::vector<double> small(N + 1, 0.0), large(N + 1, 0.0);   // sums of the c smallest / largest e_k
        if (C.ns) {
            std::vector<double> e(N, 0.0);
            for (int k = 0; k < N; ++k)
                for (int s = 0; s < C.ns; ++s) e[k] += C.c[(size_t)k * C.ns + s] * mv[s];
            std::sort(e.begin(), e.end());
            for (int c = 1; c <= N; ++c) { small[c] = small[c - 1] + e[c - 1]; large[c] = large[c - 1] + e[N - c]; }
        }
        double dlo = 1e300, dhi = -1e300;
        for (int c = 0; c <= N; ++c) {
            if (P.dmin_cnt[c] > P.dmax_cnt[c]) continue;  // empty bin
            dlo = std::min(dlo, P.dmin_cnt[c] - th * c - large[c]);
            dhi = std::max(dhi, P.dmax_cnt[c] - th * c - small[c]);
        }
        lo = dlo - dr; hi = dhi + dr;
    } else {
        for (int b = 0; b < P.B; ++b) {
            double dr = 0.0;
            double dlo = 0.0, dhi = 0.0;
            if (P.has_interaction) {
                dlo = P.dint_shared ? P.dmin_traj[0] : P.dmin_traj[b];
                dhi = P.dint_shared ? P.dmax_traj[0] : P.dmax_traj[b];
            }
            for (int k = 0; k < N; ++k) {
                dr += std::abs(C.a[(size_t)b * N + k]);
                double e = 0.0;
                for (int s = 0; s < C.ns; ++s) e += C.c[((size_t)b * N + k) * C.ns + s] * mv[s];
                const double val = -(th + e);   // diagonal of a qubit in |from>, 0 otherwise
                dlo += std::min(0.0, val); dhi += std::max(0.0, val);
            }
            dr *= std::fabs(om);
            lo = std::min(lo, dlo - dr); hi = std::max(hi, dhi + dr);
        }
    }
    centre = 0.5 * (lo + hi);
    half = std::max(0.5 * (hi - lo) * (1.0 + 1e-9), 1e-9);
}

// half-width of H at every sampling time (step-length rule, cost estimate)
static void taylor_knot_widths(Plan& P) {
    Plan::TaylorCache& C = P.tay;
    const int nt = (int)P.times.size();
    if ((int)C.w_knot.size() == nt) return;
    const int order = P.desc.interp_order;
    const PiecewiseCubic<double>& th_pc = P.tabs[0][0].det[0];
    C.w_knot.resize(nt);
    for (int i = 0; i < nt; ++i) {
        double c, hw, mv[PB200_TAYLOR_SMAX] = {};
        for (int s = 0; s < C.ns; ++s) mv[s] = eval_at(C.shape[s], P.times, P.times[i], order);
        // the spectrum of omega X does not depend on the phase of omega: |omega| bounds it
        double om = eval_at(C.om, P.times, P.times[i], order);
        if (C.phase_moves) om = std::hypot(om, eval_at(C.om_im, P.times, P.times[i], order));
        taylor_bounds(P, om, eval_at(th_pc, P.times, P.times[i], order), mv, c, hw);
        C.w_knot[i] = hw + P.diss_tay.norm;   // a master equation: + the bound of its dissipator (0 otherwise)
    }
}

// Is the Taylor propagator the cheaper choice?  (i) A cubic spline through samples of a curved function deviates from
// every smooth function by ~ |4th difference| / 384 per interval; where that floor exceeds what the fit may leave
// behind, no polynomial spans more than one sampling interval and a step costs ~10 H-applies per interval -- more than
// the Magnus path.  Worth it when at most a quarter of the intervals are like that (C2 / C5: only those at the kinks).
// (ii) Its cost is ~4.1 H-applies per unit of (spectral half-width x time) of the FULL spectrum; for very strongly
// blockaded registers the Krylov path (populated spectrum) is cheaper: limit ~12 applies per ns (C4: 7, C2: 1).
static bool taylor_worthwhile(Plan& P, double gtol) {
    const int nt = (int)P.times.size();
    if (nt < 8) return false;
    const double rate = gtol / std::max(P.times.back() - P.times.front(), 1e-30);
    const double allow = 0.25 * rate / P.n;
    std::vector<const PiecewiseCubic<double>*> pcs = {&P.tay.om, &P.tabs[0][0].det[0]};
    if (P.tay.phase_moves) pcs.push_back(&P.tay.om_im);   // a phase jump under amplitude is a kink of both parts
    for (int s = 0; s < P.tay.ns; ++s) pcs.push_back(&P.tay.shape[s]);
    std::vector<char> rough(nt, 0);
    for (const PiecewiseCubic<double>* pc : pcs) {
        const int np = pc->pieces();
        auto y = [&](int i) { return i < np ? pc->c0[i] : pc->y_last; };
        for (int i = 2; i + 2 < nt; ++i) {
            const double d4 = std::fabs(y(i + 2) - 4.0 * y(i + 1) + 6.0 * y(i) - 4.0 * y(i - 1) + y(i - 2));
            if (d4 / 384.0 > allow) rough[i] = 1;
        }
    }
    int cnt = 0;
    for (char c : rough) cnt += c;
    if (4 * cnt > nt) { g_taylor_why = "splines too rough for multi-interval polynomial steps"; return false; }
    // (iii) a master equation: the alternative is the splitting path, not Krylov; measured faster at every size it runs,
    // under a moving drive phase too (experiments/lindblad_cost.py, lindblad_phase_cost.py, DESIGN.md section 3a)
    if (P.has_diss) return true;
    taylor_knot_widths(P);
    double wsum = 0.0;
    for (int i = 0; i + 1 < nt; ++i) wsum += 0.5 * (P.tay.w_knot[i] + P.tay.w_knot[i + 1]) * (P.times[i + 1] - P.times[i]);
    const double applies_per_interval = 4.1 * wsum / std::max(nt - 1, 1);
    const double hi_mean_ns = (P.times.back() - P.times.front()) / std::max(nt - 1, 1) * 1e3;
    constexpr double kTaylorMaxAppliesPerNs = 12.0;
    const bool cheap = applies_per_interval / std::max(hi_mean_ns, 1e-30) <= kTaylorMaxAppliesPerNs;
    if (!cheap) g_taylor_why = "spectrum too wide: the Krylov path is expected to be cheaper";
    return cheap;
}

struct TaylorPoly {      // monomial coefficients in u of one coefficient function on a step, and the fit residual
    std::vector<double> c;
    double resid = 0.0;
};

// degree-p Chebyshev interpolant of the spline on [a, a+h], as monomials in u = (t-a)/h; residual on a fine grid
static TaylorPoly taylor_fit(const PiecewiseCubic<double>& pc, const std::vector<double>& x, int order, double a, double h,
                             int p) {
    typedef long double ld;
    const ld PI = 3.14159265358979323846264338327950288L;
    const int m = p + 1;
    std::vector<ld> f(m), ck(m, 0.0L);
    for (int i = 0; i < m; ++i) {
        const ld xi = cosl(PI * (2 * i + 1) / (2.0L * m));
        f[i] = (ld)eval_at(pc, x, a + h * (double)(0.5L * (xi + 1.0L)), order);
    }
    for (int k = 0; k < m; ++k) {
        ld s = 0.0L;
        for (int i = 0; i < m; ++i) s += f[i] * cosl(PI * k * (2 * i + 1) / (2.0L * m));
        ck[k] = s * (k == 0 ? 1.0L : 2.0L) / m;
    }
    // Chebyshev series in x -> monomials in x
    std::vector<ld> mono(m, 0.0L), Tm2(m, 0.0L), Tm1(m, 0.0L), Tk(m, 0.0L);
    Tm2[0] = 1.0L;                       // T_0
    mono[0] += ck[0];
    if (m > 1) { Tm1[1] = 1.0L; for (int i = 0; i < m; ++i) mono[i] += ck[1] * Tm1[i]; }
    for (int k = 2; k < m; ++k) {
        for (int i = 0; i < m; ++i) Tk[i] = (i > 0 ? 2.0L * Tm1[i - 1] : 0.0L) - Tm2[i];
        for (int i = 0; i < m; ++i) mono[i] += ck[k] * Tk[i];
        Tm2 = Tm1; Tm1 = Tk;
    }
    // x = 2u - 1
    std::vector<ld> cu(m, 0.0L), pw(m, 0.0L), nx(m, 0.0L);
    pw[0] = 1.0L;                        // (2u - 1)^0
    for (int k = 0; k < m; ++k) {
        for (int i = 0; i < m; ++i) cu[i] += mono[k] * pw[i];
        for (int i = 0; i < m; ++i) nx[i] = (i > 0 ? 2.0L * pw[i - 1] : 0.0L) - pw[i];
        pw = nx;
    }
    TaylorPoly out;
    out.c.resize(m);
    for (int i = 0; i < m; ++i) out.c[i] = (double)cu[i];
    // residual: 4 points per sampling interval inside the step (at least 9 points)
    const int ia = find_piece(x, a + 1e-15), ib = find_piece(x, a + h - 1e-15);
    const int npts = std::max(9, 4 * (ib - ia + 1) + 1);
    double r = 0.0;
    for (int q = 0; q < npts; ++q) {
        const double u = (double)q / (npts - 1);
        double pv = 0.0;
        for (int i = m - 1; i >= 0; --i) pv = pv * u + out.c[i];
        r = std::max(r, std::fabs(pv - eval_at(pc, x, a + h * u, order)));
    }
    out.resid = r;
    return out;
}

// Taylor order from the scalar majorant  y' = h m(u) y,  m(u) = sum_j m_j u^j >= |H~(u)|:  |chi_k| <= y_k with
// (k+1) y_{k+1} = h sum_j m_j y_{k-j}.  Returns the smallest K whose remainder sum_{k>K} y_k is below tol.
static int taylor_order(double h, const std::vector<double>& mj, double tol, double& tail_out) {
    const int p = (int)mj.size() - 1;
    std::vector<double> y(1, 1.0);
    const int kcap = 1200;
    for (int k = 0; k < kcap; ++k) {
        double s = 0.0;
        for (int j = 0; j <= std::min(p, k); ++j) s += mj[j] * y[k - j];
        y.push_back(h * s / (k + 1));
        if (k > 8 && y.back() < 1e-40 && y.back() < y[k]) break;
    }
    double tail = 0.0;
    int kk = (int)y.size() - 1;
    for (; kk >= 1; --kk) {
        if (tail + y[kk] > tol) break;
        tail += y[kk];
    }
    tail_out = tail;
    return std::max(kk, 1);
}

// First order k_lo of a K-order step that stores its outputs (chi_{k+1}, and G_k with g_stored) in single precision:
// the orders k >= k_lo.  A stored chi_j carries at most u32 |chi_j| <= u32 y_j of rounding, which reaches psi(1) once
// through the accumulator and again through every later order: with S_j = sum_{k=j..K} z_k of the same majorant
// recurrence started from a unit impulse at order j, at most u32 y_j S_j.  A stored G_j = X chi_j is only read by the
// history terms om_i G_j of the later orders, whose coefficients |om_i| |X| are part of m_i, so its rounding costs at
// most u32 y_j (S_j - 1).  Returns the smallest k_lo whose summed bound (*bound_out) is <= tol; K when none is.
static int taylor_lowprec_order(double h, const std::vector<double>& mj, int K, bool g_stored, double tol,
                                double& bound_out) {
    constexpr double u32 = 5.9604644775390625e-08;   // 2^-24
    const int p = (int)mj.size() - 1;
    std::vector<double> y(K + 1, 0.0), S(K + 1, 0.0), z(K + 1);
    y[0] = 1.0;
    for (int k = 0; k < K; ++k) {
        double s = 0.0;
        for (int j = 0; j <= std::min(p, k); ++j) s += mj[j] * y[k - j];
        y[k + 1] = h * s / (k + 1);
    }
    for (int j = 1; j <= K; ++j) {
        std::fill(z.begin(), z.end(), 0.0);
        z[j] = 1.0;
        double sum = 1.0;
        for (int k = j; k < K; ++k) {
            double s = 0.0;
            for (int i = 0; i <= std::min(p, k - j); ++i) s += mj[i] * z[k - i];
            z[k + 1] = h * s / (k + 1);
            sum += z[k + 1];
        }
        S[j] = sum;
    }
    // cost(L): chi_j for j = L+1 .. K, G_j for j = L .. K-2 (the last order stores no G)
    double bound = 0.0;
    int k_lo = K;
    for (int L = K - 1; L >= 0; --L) {
        double add = u32 * y[L + 1] * S[L + 1];
        if (g_stored && L <= K - 2) add += u32 * y[L] * (S[L] - 1.0);
        if (bound + add > tol) break;
        bound += add;
        k_lo = L;
    }
    bound_out = bound;
    return k_lo;
}

// One order of a Taylor step: the tiled variant that the plan and the arguments select, or the plain kernel of small
// registers (!tiled).  cplx: a step whose drive phase moves inside it
static void launch_taylor_order(const Plan& P, bool tiled, const TaylorArgs& a, bool cplx) {
    const bool diss = a.n_pair > 0;
    if (!tiled) {
        const dim3 grid((unsigned)((P.D + 255) / 256), (unsigned)P.B);
        if (diss && cplx) stage_d2_taylor_small_kernel<true, true><<<grid, 256, 0, P.stream>>>(a);
        else if (diss) stage_d2_taylor_small_kernel<false, true><<<grid, 256, 0, P.stream>>>(a);
        else if (cplx) stage_d2_taylor_small_kernel<true><<<grid, 256, 0, P.stream>>>(a);
        else stage_d2_taylor_small_kernel<false><<<grid, 256, 0, P.stream>>>(a);
        return;
    }
    // one state unless the table holds per-trajectory factors (batches); a uniform drive with detuning shapes is one state
    const bool uniform = !a.table || (a.tab_shapes && P.tay.drive_uniform);
    const bool real_g = uniform && !cplx && a.unit.y == 0.0;
    const bool shard = a.shard_bits > 0;
    const int ns = a.tab_shapes ? PB200_TAYLOR_SMAX : uniform ? 0 : 1;
    for (const TaylorVariant& v : taylor_variants()) {
        if (v.uniform != uniform || v.real_g != real_g || v.shard != shard || v.ns != ns || v.cplx != cplx ||
            v.diss != diss || v.src32 != (a.src32 != 0) || v.out32 != (a.out32 != 0))
            continue;
        launch_k(v.kernel, dim3((unsigned)(P.D >> kTaylorTileBits), uniform ? 1u : (unsigned)P.B),
                 dim3(1u << (kTaylorTileBits - v.rb)), taylor_variant_smem(v, P.n), P.stream, v.pdl, a);
        return;
    }
    fail(PB200_ERR_UNSUPPORTED, "no Taylor stage kernel for UNIFORM=%d REAL_G=%d SHARD=%d NS=%d CPLX=%d DISS=%d SRC32=%d OUT32=%d",
         uniform, real_g, shard, ns, cplx, diss, a.src32, a.out32);
}

// Geometry of the Taylor stage on the 2^L amplitudes a plan holds (L = N, or N - shard_bits on a shard): the
// register-blocked single-pass kernel on its own 2^kTaylorTileBits tile (whatever tile the Magnus stages use), the local
// bits above the tile as partner loads (tiled), or the plain kernel for small registers.  n_bits is the global N.
// False where neither applies; a shard without the single-pass geometry is refused.
static bool taylor_geometry(const Plan& P, PassGeom& geo, bool& tiled) {
    const int L = P.n - P.shard_bits;
    const std::vector<PassGeom> passes = plan_passes(L, kTaylorTileBits, kMaxExtraBits);
    if (P.shard_bits && passes.size() != 1) fail(PB200_ERR_UNSUPPORTED, "shard of 2^%d amplitudes: no single-pass geometry", L);
    geo = passes[0];
    geo.n_bits = P.n;
    tiled = passes.size() == 1 && geo.first_pass && geo.hi_bits == 0 && geo.lo_bits == kTaylorTileBits;
    return tiled || P.n <= 16;
}

// One step of the Taylor propagator as the host schedules it: the polynomial fits, the centres gamma_j, the order K and
// the ring it needs.  Everything here is decided a priori, before any launch of the step.
struct TaylorStep {
    double t = 0.0, h = 0.0;
    std::vector<double> om, th;      // monomial coefficients in u of omega, theta, M_s (trailing zeros trimmed)
    std::vector<double> m[PB200_TAYLOR_SMAX];
    int p_om = 0, p_th = 0, p = 0;
    std::vector<double> gam;         // centres of H_j
    int K = 0;
    int k_lo = 0;                    // orders k >= k_lo store chi_{k+1} and G_k in single precision (K: none)
    double phi = 0.0;                // phase of the scalar centre over the step
    int n_chi = 0, n_g = 0;          // chi ring (slot 0 = the current state), G ring (and G' ring of a complex step)
    // drive of the step: 0 real along the plan's unit; 1 real along its own unit (one phase over the step, the existing
    // kernels); 2 complex, omega = om + i omi along the plan's unit (the CPLX kernels, two gathers per order)
    int drive = 0;
    c2 unit{1.0, 0.0};
    std::vector<double> omi;
    int ring() const { return (n_chi - 1) + n_g * (drive == 2 ? 2 : 1) + 1; }   // state-sized buffers beyond the state
};

// Host half of the Taylor propagator (taylor_launch_steps is the launching half): the steps of one call
// [t_start, t_stop], one at a time (next()), with the statistics the launches do not change.  A whole state launches
// every step as soon as it is scheduled (the host fit of the next step overlaps the device work); shards schedule the
// whole call before their first launch.
struct TaylorScheduler {
    Plan& P;
    double t_stop, eps = 1e-12, gtol, rate, rho_target, fit_total, fit_spent = 0.0, round2 = 0.0;
    double t, steps_len = 0.0, t_retry_len = 0.0, A_sum, C_sum[PB200_TAYLOR_SMAX], kRoundUnit = 0.05 * 1.1102230246251565e-16;
    int order, N, nt, ns;
    bool log_steps;
    bool lowprec;   // the plan (or its shards) has single-precision stage kernels for its real-drive steps
    pb200_run_stats st{};
    struct Fit { TaylorPoly om, omi, th, m[PB200_TAYLOR_SMAX]; double om_allow = 0.0; bool ok; };

    TaylorScheduler(Plan& P_, double t_start, double t_stop_, const pb200_run_opts* o) : P(P_), t_stop(t_stop_), t(t_start) {
        const double tlo = P.times.front(), thi = P.times.back();
        gtol = taylor_default_tol(P, o);
        rate = gtol / std::max(thi - tlo, 1e-30);       // error budget per unit of time
        constexpr double kTaylorRhoMax = 14.0;
        order = P.desc.interp_order;
        N = P.n;
        nt = (int)P.times.size();
        Plan::TaylorCache& C = P.tay;
        taylor_knot_widths(P);
        // Step length: rho = h W <= kTaylorRhoMax, lowered where the fp64 cancellation of the series would eat the tolerance.  The
        // rounding error of a step grows like e^rho: ~0.05 eps e^rho measured (DESIGN.md section 3a: 6e-12 per
        // step at rho = 14, 1.4e-10 at 18), random from step to step, n ~ (int W dt) / rho steps over the whole sequence;
        // it may use a fifth of the tolerance.  At the default 1e-8 this never binds (17 > 14 for C2, C4, C5).
        rho_target = kTaylorRhoMax;
        {
            double w_total = 0.0;
            for (int i = 0; i + 1 < nt; ++i) w_total += 0.5 * (C.w_knot[i] + C.w_knot[i + 1]) * (P.times[i + 1] - P.times[i]);
            for (int it = 0; it < 3; ++it) {
                const double n_est = std::max(w_total / std::max(rho_target, 1.0), 1.0);
                rho_target = std::min(kTaylorRhoMax, std::max(4.0, std::log(0.2 * gtol / (kRoundUnit * std::sqrt(n_est)))));
            }
        }
        A_sum = std::max(C.a_sum_max, 1e-300);
        ns = C.ns;
        for (int s = 0; s < PB200_TAYLOR_SMAX; ++s) C_sum[s] = std::max(C.c_sum_max[s], 1e-300);
        // The fit error is budgeted over the call: 50 % of its share of the tolerance (10 % goes to the Taylor remainders).
        fit_total = 0.5 * rate * (t_stop - t_start);
        log_steps = env_int("PB200_TAYLOR_LOG", 0) != 0;
        PassGeom geo;
        bool tiled = false;
        lowprec = taylor_geometry(P, geo, tiled) && tiled && C.uniform;
    }

    // fit of both coefficient functions on [a, a+h] with the smallest degrees that meet the residual budget.
    // Smooth stretches fit to rounding and spend nothing, so a step may also use 2 % of what is still unspent -- this is
    // what shortens the stretches of one-interval steps around a non-smooth sample, where the not-a-knot spline rings with
    // a factor 0.268 per interval (|dH| <= (r_om + r_th) N, state error <= h |dH|).
    Fit fit_step(double a, double h, bool single_piece) {
        const Plan::TaylorCache& C = P.tay;
        Fit F; F.ok = false;
        const double budget = std::max(0.5 * rate * h, 0.02 * std::max(fit_total - fit_spent, 0.0));
        // |dH| <= r_om sum|a| + r_th N + sum_s r_Ms sum|c_s| : a third of the step's allowance each, the shapes' third
        // shared equally
        const double third = budget / (3.0 * h);
        // smallest passing degree; a candidate that spans several intervals is first tried at the highest degree so
        // that a step across a non-smooth sample is refused after one fit instead of PB200_TAYLOR_PMAX + 1
        auto one = [&](const PiecewiseCubic<double>& pc, TaylorPoly& out, double allow) {
            if (!single_piece) {
                out = taylor_fit(pc, P.times, order, a, h, PB200_TAYLOR_PMAX);
                if (out.resid > allow) return false;
            }
            for (int p = 0; p < PB200_TAYLOR_PMAX; ++p) {
                TaylorPoly f = taylor_fit(pc, P.times, order, a, h, p);
                if (f.resid <= allow || (single_piece && p >= 3)) { out = f; return true; }
            }
            if (single_piece) out = taylor_fit(pc, P.times, order, a, h, PB200_TAYLOR_PMAX);
            return true;
        };
        // a moving phase: each part of omega gets half the drive's third (|d omega| <= r_re + r_im)
        F.om_allow = third / A_sum;
        if (C.phase_moves) F.ok = one(C.om, F.om, 0.5 * F.om_allow) && one(C.om_im, F.omi, 0.5 * F.om_allow);
        else F.ok = one(C.om, F.om, F.om_allow);
        F.ok = F.ok && one(P.tabs[0][0].det[0], F.th, third / N);
        for (int s = 0; s < ns && F.ok; ++s) F.ok = one(C.shape[s], F.m[s], third / ns / C_sum[s]);
        for (int s = ns; s < PB200_TAYLOR_SMAX; ++s) { F.m[s].c.assign(1, 0.0); F.m[s].resid = 0.0; }
        return F;
    }

    // end of the longest candidate step from t (in interval i0): rho accumulated over the sampling intervals up to
    // rho_target, or the length a step cut by the rho check left behind
    double candidate_end(int i0) {
        const Plan::TaylorCache& C = P.tay;
        double b = t, acc = 0.0, cur = t;
        int i = i0;
        while (i < nt - 1) {
            const double e1 = std::min(P.times[i + 1], t_stop);
            const double w = std::max(C.w_knot[i], C.w_knot[i + 1]);
            const double need = w * (e1 - cur);
            if (acc + need > rho_target) {
                if (i == i0 || acc == 0.0) b = cur + (rho_target - acc) / std::max(w, 1e-300);  // inside the first interval
                else b = cur;
                break;
            }
            acc += need; cur = e1; b = e1; ++i;
            if (e1 >= t_stop - eps) break;
        }
        b = std::min(b, t_stop);
        if (t_retry_len > 0.0) { b = std::min(b, t + t_retry_len); t_retry_len = 0.0; }
        if (b <= t + eps) b = std::min(P.times[i0 + 1], t_stop);
        return b;
    }

    // longest step [t, b] on which every spline is a polynomial of degree <= PB200_TAYLOR_PMAX to within the budget:
    // bisection over the number of whole sampling intervals beyond the first one (a step inside one interval is a cubic:
    // exact).  b comes in as the candidate end.
    Fit longest_fit(int i0, double& b) {
        const bool single = b <= P.times[i0 + 1] + eps;
        Fit F = fit_step(t, b - t, single);
        if (F.ok || single) return F;
        int lo_keep = 0, hi_keep = find_piece(P.times, b - eps) - i0;   // lo passes (one interval), hi fails
        Fit Flo; bool have_lo = false;
        while (hi_keep - lo_keep > 1) {
            const int mid = (lo_keep + hi_keep) / 2;
            const double bm = P.times[i0 + 1 + mid];
            Fit Fm = fit_step(t, bm - t, false);
            if (Fm.ok) { lo_keep = mid; Flo = Fm; have_lo = true; } else hi_keep = mid;
        }
        b = P.times[i0 + 1 + lo_keep];
        return have_lo ? Flo : fit_step(t, b - t, lo_keep == 0);
    }

    // Drive of a step where the plan's phase moves: one phase over the step (the imaginary part after the rotation onto
    // the phase of the largest of omega(0), omega(1/2), omega(1) fits in the drive's allowance, booked as fit residual)
    // runs the real kernels with the step's own unit; otherwise the complex kernels.  Returns the drive's fit residual.
    double classify_drive(Fit& F, int& drive, c2& unit) const {
        auto coef = [](const std::vector<double>& c, size_t j) { return j < c.size() ? c[j] : 0.0; };
        auto poly = [](const std::vector<double>& c, double u) {
            double v = 0.0;
            for (int i = (int)c.size() - 1; i >= 0; --i) v = v * u + c[i];
            return v;
        };
        double best = 0.0, cph = 1.0, sph = 0.0;
        for (double u : {0.0, 0.5, 1.0}) {
            const double x = poly(F.om.c, u), y = poly(F.omi.c, u), r = std::hypot(x, y);
            if (r > best) { best = r; cph = x / r; sph = y / r; }
        }
        const size_t nc = std::max(F.om.c.size(), F.omi.c.size());
        std::vector<double> xr(nc), yr(nc);   // omega e^{-i phase}
        double ybound = 0.0;
        for (size_t j = 0; j < nc; ++j) {
            xr[j] = cph * coef(F.om.c, j) + sph * coef(F.omi.c, j);
            yr[j] = cph * coef(F.omi.c, j) - sph * coef(F.om.c, j);
            ybound += std::fabs(yr[j]);
        }
        const double r2 = F.om.resid + F.omi.resid;   // |omega - fit| <= |r_re + i r_im|
        if (r2 + ybound <= F.om_allow) {
            F.om.c = xr;
            if (cph != 1.0 || sph != 0.0) {
                const c2 u = P.tay.unit;
                drive = 1;
                unit = {u.x * cph - u.y * sph, u.x * sph + u.y * cph};
            }
            return r2 + ybound;
        }
        drive = 2;
        return r2;
    }

    // strip trailing zero coefficients (of omega's imaginary part too on a complex step); returns the shapes' degree
    static int trim(Fit& F, bool cplx) {
        auto trim1 = [](std::vector<double>& c, double scale) {
            while (c.size() > 1 && std::fabs(c.back()) <= 1e-15 * scale) c.pop_back();
        };
        double so = 0.0, sh = 0.0;
        for (double v : F.om.c) so = std::max(so, std::fabs(v));
        if (cplx) for (double v : F.omi.c) so = std::max(so, std::fabs(v));
        for (double v : F.th.c) sh = std::max(sh, std::fabs(v));
        trim1(F.om.c, std::max(so, 1e-300)); trim1(F.th.c, std::max(sh, 1e-300));
        if (cplx) trim1(F.omi.c, std::max(so, 1e-300));
        int p_m = 0;
        for (int q = 0; q < PB200_TAYLOR_SMAX; ++q) {
            double sm = 0.0;
            for (double v : F.m[q].c) sm = std::max(sm, std::fabs(v));
            trim1(F.m[q].c, std::max(sm, 1e-300));
            p_m = std::max(p_m, (int)F.m[q].c.size() - 1);
        }
        return p_m;
    }

    // centres gamma_j and norm bounds m_j of H_j, j <= p
    void centres_and_bounds(const Fit& F, bool cplx, int p_om, int p, std::vector<double>& gam, std::vector<double>& mj) const {
        auto th_c = [&](int j) { return j < (int)F.th.c.size() ? F.th.c[j] : 0.0; };
        auto m_c = [&](int q, int j) { return j < (int)F.m[q].c.size() ? F.m[q].c[j] : 0.0; };
        // |omega_j|: the spectrum of omega_j X does not depend on the phase of omega_j
        auto om_abs = [&](int j) {
            const double x = j < (int)F.om.c.size() ? F.om.c[j] : 0.0;
            if (!cplx) return std::fabs(x);
            return std::hypot(x, j < (int)F.omi.c.size() ? F.omi.c[j] : 0.0);
        };
        gam.assign(p + 1, 0.0); mj.assign(p + 1, 0.0);
        double c0, hw0, mv[PB200_TAYLOR_SMAX];
        for (int q = 0; q < PB200_TAYLOR_SMAX; ++q) mv[q] = m_c(q, 0);
        taylor_bounds(P, cplx ? om_abs(0) : F.om.c[0], F.th.c[0], mv, c0, hw0);
        // the dissipator is static and not centred: its bound joins m_0 (0 without one)
        gam[0] = c0; mj[0] = hw0 + P.diss_tay.norm;
        for (int j = 1; j <= p; ++j) {
            const double thj = th_c(j), omj = j <= p_om ? om_abs(j) : 0.0;
            gam[j] = -thj * 0.5 * N;
            double mm = 0.0;
            for (int q = 0; q < ns; ++q) mm += std::fabs(m_c(q, j)) * C_sum[q];
            mj[j] = std::fabs(thj) * 0.5 * N + mm + std::fabs(omj) * A_sum;
        }
    }

    // the order of step s, its log line and its share of the error estimate; rho = h sum_j m_j / (j + 1)
    void record(TaylorStep& s, const Fit& F, const std::vector<double>& mj, int p_m, double om_resid, double rho) {
        double trunc_bound = 0.0, round32 = 0.0;
        s.K = taylor_order(s.h, mj, std::max(1e-15, 0.1 * rate * s.h), trunc_bound);
        // the tail orders in single precision: another 10 % of the step's share of the tolerance
        s.k_lo = (lowprec && s.drive != 2) ? taylor_lowprec_order(s.h, mj, s.K, s.n_g > 0, 0.1 * rate * s.h, round32) : s.K;
        st.n_applies += s.K; st.n_exponentials += 1; ++st.n_steps;
        if (log_steps)
            fprintf(stderr, "taylor step t=%.6f h_ns=%.3f p_om=%d p_th=%d p_m=%d K=%d ring=%d rho=%.3f resid=%.2e/%.2e/%.2e drive=%s k_lo=%d\n",
                    s.t, s.h * 1e3, s.p_om, s.p_th, p_m, s.K, s.ring() + 1, mj[0] * s.h, om_resid, F.th.resid, F.m[0].resid,
                    s.drive == 2 ? "cplx" : s.drive == 1 ? "rot" : "real", s.k_lo);
        st.max_rho = std::max(st.max_rho, rho);
        double fit_m = 0.0;
        for (int q = 0; q < ns; ++q) fit_m += C_sum[q] * F.m[q].resid;
        const double fit_err = s.h * (A_sum * om_resid + N * F.th.resid + fit_m);
        st.err_estimate += trunc_bound + round32 + fit_err;
        fit_spent += fit_err;
        { const double r = kRoundUnit * std::exp(std::min(rho, 40.0)); round2 += r * r; }
        steps_len += s.h;
    }

    // the next step of the call; false once t_stop is reached
    bool next(TaylorStep& s) {
        while (t < t_stop - eps) {
            const int i0 = find_piece(P.times, t + eps);
            double b = candidate_end(i0);
            Fit F = longest_fit(i0, b);
            const double h = b - t;
            int drive = 0;
            c2 unit = P.tay.unit;
            const double om_resid = P.tay.phase_moves ? classify_drive(F, drive, unit) : F.om.resid;
            const int p_m = trim(F, drive == 2);
            const int p_om = std::max((int)F.om.c.size(), drive == 2 ? (int)F.omi.c.size() : 0) - 1;
            const int p_th = std::max((int)F.th.c.size() - 1, p_m);   // degree of the diagonal (own-element) history
            const int p = std::max(p_om, p_th);
            std::vector<double> gam, mj;
            centres_and_bounds(F, drive == 2, p_om, p, gam, mj);
            // the fp64 cancellation of the series grows like e^rho: a step whose majorant exponent overshoots the target
            // (the half-width grew inside the step) is cut and fitted again
            double rho = 0.0;
            for (int j = 0; j <= p; ++j) rho += mj[j] / (j + 1);
            rho *= h;
            if (rho > 1.12 * rho_target && h > 1e-9) {
                t_retry_len = h * rho_target / rho;
                continue;
            }
            s.t = t; s.h = h;
            s.om = F.om.c; s.th = F.th.c;
            for (int q = 0; q < PB200_TAYLOR_SMAX; ++q) s.m[q] = F.m[q].c;
            s.p_om = p_om; s.p_th = p_th; s.p = p;
            s.gam = gam;
            s.n_chi = p_th + 2;
            s.n_g = p_om >= 1 ? p_om + 1 : 0;
            s.drive = drive; s.unit = unit;
            s.omi = drive == 2 ? F.omi.c : std::vector<double>();
            // phase of the scalar centre: exp(-i h int_0^1 sum_j gam_j u^j du)
            double phi = 0.0;
            for (int j = 0; j <= p; ++j) phi += gam[j] / (j + 1);
            s.phi = phi * h;
            record(s, F, mj, p_m, om_resid, rho);
            t = b;
            return true;
        }
        return false;
    }

    // statistics of the whole call (gpu_ms and n_launches come from the launching half)
    pb200_run_stats finish(double gpu_ms, long long launches) const {
        pb200_run_stats out = st;
        out.gpu_ms = gpu_ms;
        out.n_launches = launches;
        const double hi_mean = (P.times.back() - P.times.front()) / std::max(nt - 1, 1);
        out.mean_step_samples = out.n_steps ? steps_len / out.n_steps / hi_mean : 0.0;
        out.err_estimate += std::sqrt(round2);
        out.integrator = 3;
        return out;
    }
};

// Ring of one step: chi[0] = the current state, the other slots from the buffers that are not the state (the Magnus
// aux buffers too when the plan has them), then the plan's own Taylor work buffers, allocated on first need.
struct TaylorRing {
    std::vector<c2*> chi, gr, gr2;   // gr2: G' of a complex step
    DevBuf<c2>* acc_slot = nullptr;
};

static void taylor_grow_ring(Plan& P, int need) {
    int have = 2 + (P.aux[0] ? 6 : 0) + (int)P.tay_ws.size();
    while (have < need) {
        P.tay_ws.emplace_back(P, (size_t)P.D * P.B);
        ++have;
    }
}

static TaylorRing taylor_ring(Plan& P, const TaylorStep& s) {
    std::vector<DevBuf<c2>*> free_slots;
    for (int i = 0; i < 3; ++i) if (i != P.cur) free_slots.push_back(&P.buf[i]);
    if (P.aux[0]) for (int i = 0; i < 6; ++i) free_slots.push_back(&P.aux[i]);
    taylor_grow_ring(P, s.ring());
    for (size_t i = 0; i < P.tay_ws.size(); ++i) free_slots.push_back(&P.tay_ws[i]);
    TaylorRing R;
    R.chi.resize(s.n_chi); R.gr.resize(s.n_g); R.gr2.resize(s.drive == 2 ? s.n_g : 0);
    int fs = 0;
    R.chi[0] = P.buf[P.cur].get();
    for (int i = 1; i < s.n_chi; ++i) R.chi[i] = free_slots[fs++]->get();
    for (int i = 0; i < s.n_g; ++i) R.gr[i] = free_slots[fs++]->get();
    for (size_t i = 0; i < R.gr2.size(); ++i) R.gr2[i] = free_slots[fs++]->get();
    R.acc_slot = free_slots[fs++];
    return R;
}

// the arguments of a Taylor stage that depend on the plan alone: chi_k = v and chi_{k+1} = out, the interaction, the
// per-trajectory table, the drive's states and unit, the shard.  Everything else is zero: scale, history, accumulator
static TaylorArgs taylor_plan_args(const Plan& P, const PassGeom& geo, const c2* v, c2* out, c2 unit) {
    TaylorArgs a{};
    a.v = v; a.out = out;
    a.dint = P.has_interaction ? P.dint.get() : nullptr;
    a.dint_stride = P.dint_shared ? 0 : P.D;
    a.cpl = P.has_interaction ? P.cpl.get() : nullptr;
    a.cpl_stride = P.dint_shared ? 0 : (long long)P.n * P.n;
    a.ryd_bit = P.desc.rydberg_state;
    a.D = P.D;
    a.geo = geo;
    a.unit = unit;
    a.table = P.tay.uniform ? nullptr : P.tay.d_tab.get();
    a.tab_shapes = P.tay.tab_shapes;
    a.to_bit = P.desc.drives[0].state_to; a.from_is_one = P.desc.drives[0].state_from;
    a.shard_bits = P.shard_bits; a.shard = P.shard;
    if (P.has_diss) {
        for (int i = 0; i < 4; ++i) { a.dw[i] = P.diss_tay.dw[i]; a.df[i] = P.diss_tay.df[i]; }
        a.n_pair = P.n / 2;
        a.diss_flip = P.diss_tay.flip ? 1 : 0;
    }
    return a;
}

// arguments of order k of a step
static TaylorArgs taylor_args(const Plan& P, const PassGeom& geo, const TaylorStep& s, const TaylorRing& R, int k) {
    auto th_c = [&](int j) { return j < (int)s.th.size() ? s.th[j] : 0.0; };
    auto m_c = [&](int q, int j) { return j < (int)s.m[q].size() ? s.m[q][j] : 0.0; };
    TaylorArgs a = taylor_plan_args(P, geo, R.chi[k % s.n_chi], R.chi[(k + 1) % s.n_chi], s.unit);
    a.g_out = (s.n_g && k + 1 < s.K) ? R.gr[k % s.n_g] : nullptr;
    a.acc = R.acc_slot->get();
    a.th0 = s.th[0]; a.gam0 = s.gam[0]; a.om0 = s.om[0];
    for (int q = 0; q < PB200_TAYLOR_SMAX; ++q) a.m0[q] = m_c(q, 0);
    a.scale = {0.0, -s.h / (k + 1)};
    a.src32 = k > s.k_lo;
    a.out32 = k >= s.k_lo;
    a.nh = std::min(s.p, k);
    for (int j = 1; j <= a.nh; ++j) {
        const double thj = th_c(j), omj = j < (int)s.om.size() ? s.om[j] : 0.0;
        bool any_m = false;
        for (int q = 0; q < PB200_TAYLOR_SMAX; ++q) { a.hm[q][j - 1] = m_c(q, j); any_m = any_m || a.hm[q][j - 1] != 0.0; }
        a.hth[j - 1] = thj; a.hgam[j - 1] = s.gam[j]; a.hom[j - 1] = omj;
        a.hchi[j - 1] = (thj != 0.0 || any_m || s.gam[j] != 0.0) ? R.chi[(k - j) % s.n_chi] : nullptr;
        a.hg[j - 1] = (omj != 0.0) ? R.gr[(k - j) % s.n_g] : nullptr;
        // chi_{k-j} was written by order k-j-1, G_{k-j} by order k-j
        if (k - j - 1 >= s.k_lo) a.hchi32 |= 1u << (j - 1);
        if (k - j >= s.k_lo) a.hg32 |= 1u << (j - 1);
        if (s.drive == 2) {
            const double omij = j < (int)s.omi.size() ? s.omi[j] : 0.0;
            a.homi[j - 1] = omij;
            a.hg2[j - 1] = (omij != 0.0) ? R.gr2[(k - j) % s.n_g] : nullptr;
        }
    }
    if (s.drive == 2) {
        a.om0i = s.omi[0];
        a.g2_out = (s.n_g && k + 1 < s.K) ? R.gr2[k % s.n_g] : nullptr;
    }
    const bool last = (k + 1 == s.K);
    // sum_k chi_k: the update of order k adds chi_{k+1} and, with acc_add_v, chi_k.  Where every order k >= 1 reads
    // chi_{k-1} as a history term, the update takes it too, and the accumulator is read and written on every third
    // order only: order 0 writes chi_0 + chi_1, order k = 0 mod 3 adds chi_{k-1} + chi_k + chi_{k+1}, and the last
    // order adds what is left.  Otherwise every even order adds chi_k + chi_{k+1}.
    bool chi_hist = false;   // hchi[0] is set on every order k >= 1
    if (s.p >= 1) {
        chi_hist = th_c(1) != 0.0 || s.gam[1] != 0.0;
        for (int q = 0; q < PB200_TAYLOR_SMAX; ++q) chi_hist = chi_hist || m_c(q, 1) != 0.0;
    }
    const int period = chi_hist ? 3 : 2;
    a.acc_read = k > 0;
    if (k % period == 0) { a.acc_on = 1; a.acc_add_v = 1; a.acc_add_h = k > 0 && chi_hist; }
    else { a.acc_on = last ? 1 : 0; a.acc_add_v = k % period == 2; a.acc_add_h = 0; }
    a.acc_mul = last ? c2{std::cos(s.phi), -std::sin(s.phi)} : c2{1.0, 0.0};
    return a;
}

// CUDA events of a group of plans, one per plan, released on every exit path
struct ShardEvents {
    std::vector<cudaEvent_t> ev;
    ShardEvents(const std::vector<Plan*>& G, unsigned flags) : ev(G.size(), nullptr) {
        for (size_t r = 0; r < G.size(); ++r) {
            CUDA_CHECK(cudaSetDevice(G[r]->desc.device));
            CUDA_CHECK(cudaEventCreateWithFlags(&ev[r], flags));
        }
    }
    ~ShardEvents() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
    ShardEvents(const ShardEvents&) = delete;
    ShardEvents& operator=(const ShardEvents&) = delete;
};

// Launching half of the Taylor propagator for the plans that hold one state: {&P}, or the linked shards in shard order.
// next(s) yields the steps of the call.  Returns the largest device time of any plan, in ms.  On shards, order k on
// shard r reads chi_k of its peers: it waits for the previous launch (order k - 1, or the last order of the previous
// step) of every peer, and every shard's waits for an order are enqueued before any shard records that order's event.
// A slot a peer may still be gathering from is never overwritten: n_chi >= 2, and every order waits for the one before
// it.  The previous call ended with every stream synchronised.  A whole state records no event per order, so
// programmatic dependent launch chains its orders.
template <class Next>
static float taylor_launch_steps(const std::vector<Plan*>& G, const PassGeom& geo, bool tiled, Next&& next,
                                 long long& launches) {
    const int count = (int)G.size(), sb = count > 1 ? G[0]->shard_bits : 0;   // a whole state has no peers
    // plan r, its device current (a whole state's already is)
    auto use = [&](int r) -> Plan& {
        if (count > 1) CUDA_CHECK(cudaSetDevice(G[r]->desc.device));
        return *G[r];
    };
    ShardEvents order_ev(sb ? G : std::vector<Plan*>(), cudaEventDisableTiming), t0(G, cudaEventDefault),
        t1(G, cudaEventDefault);
    for (int r = 0; r < count; ++r) CUDA_CHECK(cudaEventRecord(t0.ev[r], use(r).stream));
    bool first = true;
    std::vector<TaylorRing> R(count);
    std::deque<std::vector<double>> tables;   // tables of rotated steps, until the call's last synchronisation
    for (TaylorStep s; next(s);) {
        for (int r = 0; r < count; ++r) {
            Plan& P = use(r);
            R[r] = taylor_ring(P, s);
            taylor_table_unit(P, s.drive == 1 ? s.unit : P.tay.unit, tables);
        }
        for (int k = 0; k < s.K; ++k) {
            for (int r = 0; r < count; ++r) {
                Plan& P = use(r);
                TaylorArgs a = taylor_args(P, geo, s, R[r], k);
                for (int q = 0; q < sb; ++q) {
                    const int peer = r ^ (1 << q);
                    a.peer[q] = R[peer].chi[k % s.n_chi];
                    if (!first) CUDA_CHECK(cudaStreamWaitEvent(P.stream, order_ev.ev[peer], 0));
                }
                launch_taylor_order(P, tiled, a, s.drive == 2);
                ++launches;
            }
            for (int r = 0; r < count && sb; ++r) CUDA_CHECK(cudaEventRecord(order_ev.ev[r], use(r).stream));
            first = false;
        }
        CUDA_CHECK(cudaGetLastError());
        // the accumulator becomes the current state buffer
        for (int r = 0; r < count; ++r) std::swap(G[r]->buf[G[r]->cur], *R[r].acc_slot);
    }
    float ms_max = 0.f;
    for (int r = 0; r < count; ++r) CUDA_CHECK(cudaEventRecord(t1.ev[r], use(r).stream));
    for (int r = 0; r < count; ++r) {
        CUDA_CHECK(cudaEventSynchronize(t1.ev[r]));
        float ms = 0.f;
        CUDA_CHECK(cudaEventElapsedTime(&ms, t0.ev[r], t1.ev[r]));
        ms_max = std::max(ms_max, ms);
    }
    return ms_max;
}

// a whole state: each step is launched as soon as it is scheduled, so the host fit of the next step overlaps the device
static void propagate_taylor(Plan& P, double t_start, double t_stop, const pb200_run_opts* o, pb200_run_stats* stats) {
    PassGeom geo;
    bool tiled = false;
    if (!taylor_geometry(P, geo, tiled)) fail(PB200_ERR_UNSUPPORTED, "Taylor propagator: unsupported register size");
    ensure_aux_buffers(P);
    TaylorScheduler S(P, t_start, t_stop, o);
    long long launches = 0;
    const float ms = taylor_launch_steps({&P}, geo, tiled, [&S](TaylorStep& s) { return S.next(s); }, launches);
    if (stats) *stats = S.finish(ms, launches);
}

// H(t) parameters as an "exponential" description with w = 1 (for apply_h)
static ExpParams params_at(const Plan& P, double t) {
    ExpParams E;
    const int N = P.n, B = P.B, nd = P.n_drives;
    E.g.assign((size_t)B * nd * N, cplx(0)); E.th.assign((size_t)B * nd * N, 0.0); E.w = 1.0;
    if (P.has_slm) E.wc = eval_at(P.slm_coef, P.times, t, P.desc.interp_order);
    for (int tr = 0; tr < B; ++tr)
        for (int q = 0; q < nd; ++q) {
            const DriveTables& T = P.tabs[tr][q];
            const int rows = (int)T.coef.size();
            for (int k = 0; k < N; ++k) {
                const int r = rows == 1 ? 0 : k;
                E.g[pidx(P, tr, q, k)] = eval_at(T.coef[r], P.times, t, P.desc.interp_order);
                E.th[pidx(P, tr, q, k)] = eval_at(T.det[r], P.times, t, P.desc.interp_order);
            }
        }
    return E;
}

// one plain H(t)-apply as a stage: H(t) unscaled (rho = 1, gamma0 = 0) in the device table and in the uniform drive
struct ApplyH {
    bool uniform, real_g;
    UniformDrive ud{};
    std::vector<PassGeom> passes;

    void launch(Plan& P, const c2* in, c2* out, long long& launches) const {
        launch_stage(P, passes, in, nullptr, nullptr, out, StageCoef{{0, 0}, {0, 0}, {1, 0}}, uniform, real_g, ud,
                     P.d_table.get(), launches);
    }
};

// out = H(t) in (device buffers [B][D]); returns the set-up, which stays valid until the device table is rewritten
static ApplyH apply_h_device(Plan& P, double t, const c2* in, c2* out, long long& launches) {
    const ExpParams E = params_at(P, t);
    double gamma0, rho; std::vector<double> host;
    build_tables(P, E, gamma0, rho, host, is_d2path(P), /*scaled=*/false);
    ensure_table_capacity(P, host.size());
    CUDA_CHECK(cudaMemcpyAsync(P.d_table.get(), host.data(), host.size() * sizeof(double), cudaMemcpyHostToDevice, P.stream));
    CUDA_CHECK(cudaStreamSynchronize(P.stream));
    ApplyH A;
    A.uniform = one_uniform_state(P);
    A.real_g = E.g[0].imag() == 0.0;
    A.ud.g = {E.g[0].real(), E.g[0].imag()}; A.ud.theta = E.th[0]; A.ud.w = 1.0; A.ud.gamma = 0.0;
    A.passes = plan_passes(P.n, kStageTileBits, kMaxExtraBits);
    A.launch(P, in, out, launches);
    CUDA_CHECK(cudaGetLastError());
    return A;
}

}  // namespace pb200

// ===========================================================================
// C ABI
// ===========================================================================
using namespace pb200;

struct pb200_plan {
    Plan p;
};

// entry points that act on a whole state through one plan: a shard only holds a slice
static void refuse_shard(const Plan& P, const char* who, const char* instead) {
    if (P.shard_bits)
        fail(PB200_ERR_STATE, "%s: the plan is shard %d of %d of a state; use %s on the linked shards", who, P.shard,
             1 << P.shard_bits, instead);
}

// ---- state-vector shards -------------------------------------------------------------------------------------------
// A shard is an ordinary plan holding 2^L amplitudes (L = N - shard_bits) of one state: the global indices
// [shard 2^L, (shard + 1) 2^L).  One process drives every shard of a group: the host schedule of a call is computed
// once, then every order of the Taylor series is launched on every shard (taylor_launch_steps), whose partners
// across a shard bit are loads from the peer's chi_k (peer access between distinct devices).

// plans[i] = shard i of a group linked by pb200_shards_link
static std::vector<Plan*> shard_group(pb200_plan** plans, int count, const char* who) {
    if (!plans || count < 2) fail(PB200_ERR_INVALID, "%s: pass the plans of every shard", who);
    std::vector<Plan*> G(count);
    for (int i = 0; i < count; ++i) {
        if (!plans[i]) fail(PB200_ERR_INVALID, "%s: null plan", who);
        G[i] = &plans[i]->p;
    }
    for (int i = 0; i < count; ++i)
        if (G[i]->group != G)
            fail(PB200_ERR_STATE, "%s: plans[] is not a linked shard group in shard order (pb200_shards_link)", who);
    return G;
}

static void shards_sync(const std::vector<Plan*>& G) {
    for (Plan* P : G) {
        CUDA_CHECK(cudaSetDevice(P->desc.device));
        CUDA_CHECK(cudaStreamSynchronize(P->stream));
    }
}

// out_r = H(t) in_r on every shard: the sharded stage with scale 1, no history and the accumulator off computes
// (Dint - theta n_from + omega X) v.  The inputs are complete (every stream synchronised) before any shard reads a peer's.
static void shards_apply_h(const std::vector<Plan*>& G, double t, const std::vector<c2*>& in, const std::vector<c2*>& out) {
    const Plan& P0 = *G[0];
    PassGeom geo;
    bool tiled = false;
    taylor_geometry(P0, geo, tiled);
    const int order = P0.desc.interp_order;
    const double om = eval_at(P0.tay.om, P0.times, t, order), th = eval_at(P0.tabs[0][0].det[0], P0.times, t, order);
    const bool cplx = P0.tay.phase_moves;
    shards_sync(G);
    const int count = (int)G.size();
    std::deque<std::vector<double>> tables;
    for (int r = 0; r < count; ++r) {
        Plan& P = *G[r];
        CUDA_CHECK(cudaSetDevice(P.desc.device));
        taylor_table_unit(P, P.tay.unit, tables);
        TaylorArgs a = taylor_plan_args(P, geo, in[r], out[r], P.tay.unit);
        if (cplx) a.om0i = eval_at(P0.tay.om_im, P0.times, t, order);
        for (int s = 0; s < P.tay.ns; ++s) a.m0[s] = eval_at(P.tay.shape[s], P.times, t, order);
        a.th0 = th; a.om0 = om;
        a.scale = {1.0, 0.0};
        a.acc_mul = {1.0, 0.0};
        for (int q = 0; q < P.shard_bits; ++q) a.peer[q] = in[r ^ (1 << q)];
        launch_taylor_order(P, tiled, a, cplx);
    }
    CUDA_CHECK(cudaGetLastError());
    shards_sync(G);
}

// ---- expectation of an operator given as monomial terms (pb200_state_expect / pb200_shards_expect) -----------------
// argument checks of an operator on n qudits of dimension dim; no device call
static void check_op_terms(const pb200_op_terms* op, int n, int dim, const char* who) {
    if (!op) fail(PB200_ERR_INVALID, "%s: null operator", who);
    if (op->n_terms < 0) fail(PB200_ERR_INVALID, "%s: n_terms = %d", who, op->n_terms);
    if (op->n_terms == 0) return;
    if (!op->coeff || !op->site_start) fail(PB200_ERR_INVALID, "%s: null coeff or site_start", who);
    if (op->site_start[0] != 0) fail(PB200_ERR_INVALID, "%s: site_start[0] = %d, must be 0", who, op->site_start[0]);
    for (int t = 0; t < op->n_terms; ++t)
        if (op->site_start[t + 1] < op->site_start[t]) fail(PB200_ERR_INVALID, "%s: site_start decreases at term %d", who, t);
    if (op->site_start[op->n_terms] > 0 && (!op->site || !op->shift || !op->weight))
        fail(PB200_ERR_INVALID, "%s: null site, shift or weight", who);
    for (int t = 0; t < op->n_terms; ++t) {
        unsigned long long seen = 0;
        for (int e = op->site_start[t]; e < op->site_start[t + 1]; ++e) {
            const int k = op->site[e], m = op->shift[e];
            if (k < 0 || k >= n) fail(PB200_ERR_INVALID, "%s: term %d names qudit %d of a %d-qudit register", who, t, k, n);
            if ((seen >> k) & 1ull) fail(PB200_ERR_INVALID, "%s: term %d names qudit %d twice", who, t, k);
            seen |= 1ull << k;
            if (m < 0 || m >= dim) fail(PB200_ERR_INVALID, "%s: term %d: shift %d outside [0, %d)", who, t, m, dim);
        }
    }
}

// host image of an operator's device table: terms, their site entries and the chunk bounds of the kernels' staging
struct ExpHost {
    bool d2 = true;
    std::vector<char> img;                 // terms | sites | chunk_t | chunk_s, each 256-byte aligned
    size_t off_sites = 0, off_ct = 0, off_cs = 0;
    int n_chunks = 0;
    unsigned used_shard_bits = 0;          // d = 2: bit x set when some mask flips shard bits x (f >> local_bits)
};

// cut the terms (sorted as the kernel reads them) into chunks of at most kExpChunkTerms terms and kExpChunkSites site
// entries; a term's site offset s0 is relative to its chunk
template <typename TermT, typename SiteT>
static void exp_pack(std::vector<std::pair<TermT, std::vector<SiteT>>>& B, ExpHost& H) {
    std::vector<TermT> T;
    std::vector<SiteT> S;
    std::vector<int> ct{0}, cs{0};
    int nt = 0, ns = 0;
    for (auto& b : B) {
        if (nt == kExpChunkTerms || ns + (int)b.second.size() > kExpChunkSites) {
            ct.push_back((int)T.size()); cs.push_back((int)S.size());
            nt = ns = 0;
        }
        b.first.s0 = ns; b.first.sn = (int)b.second.size();
        T.push_back(b.first);
        S.insert(S.end(), b.second.begin(), b.second.end());
        ++nt; ns += (int)b.second.size();
    }
    if (nt) { ct.push_back((int)T.size()); cs.push_back((int)S.size()); }
    H.n_chunks = (int)ct.size() - 1;
    auto al = [](size_t x) { return (x + 255) & ~(size_t)255; };
    H.off_sites = al(sizeof(TermT) * T.size());
    H.off_ct = H.off_sites + al(sizeof(SiteT) * S.size());
    H.off_cs = H.off_ct + al(sizeof(int) * ct.size());
    H.img.assign(H.off_cs + sizeof(int) * cs.size(), 0);
    if (!T.empty()) std::memcpy(H.img.data(), T.data(), sizeof(TermT) * T.size());
    if (!S.empty()) std::memcpy(H.img.data() + H.off_sites, S.data(), sizeof(SiteT) * S.size());
    std::memcpy(H.img.data() + H.off_ct, ct.data(), sizeof(int) * ct.size());
    std::memcpy(H.img.data() + H.off_cs, cs.data(), sizeof(int) * cs.size());
}

// d = 2: each site folds into the masks of expect_terms_d2_kernel; terms sorted by flip mask.  local_bits: index bits
// held by one plan (N for a whole state)
static ExpHost exp_host_d2(const pb200_op_terms* op, int n, int local_bits) {
    std::vector<std::pair<ExpD2Term, std::vector<ExpGenSite>>> B;
    const cplx* co = reinterpret_cast<const cplx*>(op->coeff);
    const cplx* w = reinterpret_cast<const cplx*>(op->weight);
    for (int t = 0; t < op->n_terms; ++t) {
        ExpD2Term T{};
        std::vector<ExpGenSite> gen;
        cplx c = co[t];
        for (int e = op->site_start[t]; e < op->site_start[t + 1] && c != 0.0; ++e) {
            const unsigned long long bit = 1ull << (n - 1 - op->site[e]);
            const cplx w0 = w[2 * e], w1 = w[2 * e + 1];
            if (op->shift[e]) T.f |= bit;
            if (w0 == 0.0) { T.care |= bit; T.val |= bit; c *= w1; }    // needs digit 1 (c = 0 when w1 = 0 too)
            else if (w1 == 0.0) { T.care |= bit; c *= w0; }             // needs digit 0
            else {
                c *= w0;
                const cplx r = w1 / w0;
                if (r == -1.0) T.z |= bit;
                else if (r != 1.0) gen.push_back({{r.real(), r.imag()}, bit});
            }
        }
        if (c == 0.0) continue;
        T.c = {c.real(), c.imag()};
        B.emplace_back(T, std::move(gen));
    }
    std::stable_sort(B.begin(), B.end(), [](const auto& x, const auto& y) { return x.first.f < y.first.f; });
    ExpHost H;
    for (const auto& b : B) H.used_shard_bits |= 1u << (unsigned)(b.first.f >> local_bits);
    exp_pack(B, H);
    return H;
}

// d = 3 / 4: strides of the digits, weights padded to 4
static ExpHost exp_host_general(const pb200_op_terms* op, int n, int dim) {
    std::vector<std::pair<ExpTerm, std::vector<ExpSite>>> B;
    const cplx* co = reinterpret_cast<const cplx*>(op->coeff);
    const cplx* w = reinterpret_cast<const cplx*>(op->weight);
    for (int t = 0; t < op->n_terms; ++t) {
        if (co[t] == 0.0) continue;
        ExpTerm T{};
        T.c = {co[t].real(), co[t].imag()};
        std::vector<ExpSite> sites;
        for (int e = op->site_start[t]; e < op->site_start[t + 1]; ++e) {
            ExpSite S{};
            S.stride = 1;
            for (int j = op->site[e] + 1; j < n; ++j) S.stride *= dim;
            S.shift = op->shift[e];
            for (int a = 0; a < dim; ++a) S.w[a] = {w[(size_t)e * dim + a].real(), w[(size_t)e * dim + a].imag()};
            sites.push_back(S);
        }
        B.emplace_back(T, std::move(sites));
    }
    ExpHost H;
    H.d2 = false;
    exp_pack(B, H);
    return H;
}

static ExpHost exp_host(const pb200_op_terms* op, int n, int dim, int local_bits) {
    return dim == 2 ? exp_host_d2(op, n, local_bits) : exp_host_general(op, n, dim);
}

// the device copy of an ExpHost on one plan's device
static DevBuf<char> upload_exp(const ExpHost& H, const Plan& P) {
    DevBuf<char> X(P, H.img.size());
    CUDA_CHECK(cudaMemcpyAsync(X.get(), H.img.data(), H.img.size(), cudaMemcpyHostToDevice, P.stream));
    return X;
}

// acc[2 c] += <psi_c| op |psi_c> for `count` trajectories of D amplitudes; src.p[src.shard] + c D is trajectory c
// (d = 2), psi (d > 2); X = the device copy of H.  RHO: Tr(op rho_c) of density matrices of D^2 entries instead
template <bool RHO>
static void launch_expect(const Plan& P, long long D, const ExpHost& H, const char* X, const ExpSrc& src, const c2* psi,
                          int count, double* d_acc) {
    const long long blocks = std::min<long long>((D + 255) / 256, (long long)P.sm_count * 8);
    const dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)count);
    const int* ct = reinterpret_cast<const int*>(X + H.off_ct);
    const int* cs = reinterpret_cast<const int*>(X + H.off_cs);
    if (H.d2)
        expect_terms_d2_kernel<RHO><<<grid, 256, 0, P.stream>>>(src, D, reinterpret_cast<const ExpD2Term*>(X),
                                                           reinterpret_cast<const ExpGenSite*>(X + H.off_sites), ct, cs,
                                                           H.n_chunks, d_acc);
    else
        expect_terms_kernel<RHO><<<grid, 256, 0, P.stream>>>(psi, D, P.dim, reinterpret_cast<const ExpTerm*>(X),
                                                        reinterpret_cast<const ExpSite*>(X + H.off_sites), ct, cs,
                                                        H.n_chunks, d_acc);
}

// occ[count][n] of `count` trajectories at src (RHO: density matrices of D^2 entries) of D basis states: the `rows`
// of them from basis state `off` on (rows = D, off = the shard offset, but on a density-matrix shard; basis_weight)
template <bool RHO>
static void reduce_occupation(const Plan& P, const c2* src, long long D, long long rows, long long off, int n, int count,
                              int digit, double* occ) {
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    DevBuf<double> d_occ(P, (size_t)count * n);
    const long long blocks = std::min<long long>((rows + 255) / 256, (long long)P.sm_count * 4);
    dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)count);
    device_sum(P, d_occ.get(), d_occ.size(), occ, [&] {
        occupation_kernel<RHO><<<grid, 256, sizeof(double) * n, P.stream>>>(src, d_occ.get(), D, rows, n, P.dim, digit, off);
    });
}

// corr[count][n][n] (symmetric) of `count` trajectories at src, as reduce_occupation
template <bool RHO>
static void reduce_correlation(const Plan& P, const c2* src, long long D, long long rows, long long off, int n, int count,
                               int digit, double* corr) {
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    const size_t nn = (size_t)n * n;
    DevBuf<double> d_c(P, count * nn);
    const long long blocks = std::min<long long>((rows + 2047) / 2048, (long long)P.sm_count * 4);
    dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)count);
    device_sum(P, d_c.get(), d_c.size(), corr, [&] {
        correlation_kernel<RHO><<<grid, 256, 0, P.stream>>>(src, d_c.get(), D, rows, n, P.dim, digit, off);
    });
    for (int c = 0; c < count; ++c)  // the kernel fills i <= j
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < i; ++j) corr[c * nn + (size_t)i * n + j] = corr[c * nn + (size_t)j * n + i];
}

// Bitstring shots of one state (RHO: of one density matrix's diagonal) of D basis states on n qudits, `rows` of them from
// basis state `off` on (reduce_occupation): the weights of the 2^nbits bitstrings, their inclusive prefix sum and one
// binary search per uniform (pb200_state_sample).
template <bool RHO>
static void sample_bitstrings(const Plan& P, const c2* src, long long D, long long rows, long long off, int n, int nbits,
                              int one_digit, const double* uniforms, int n_shots, int64_t* out) {
    if (nbits > 30) fail(PB200_ERR_UNSUPPORTED, "bitstring sampling: at most 30 qudits (32-bit item count of the prefix scan)");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    const long long M = 1LL << nbits;
    DevBuf<double> d_w(P, (size_t)M), d_u(P, (size_t)n_shots);
    DevBuf<long long> d_idx(P, (size_t)n_shots);
    CUDA_CHECK(cudaMemsetAsync(d_w.get(), 0, sizeof(double) * (size_t)M, P.stream));
    CUDA_CHECK(cudaMemcpyAsync(d_u.get(), uniforms, sizeof(double) * (size_t)n_shots, cudaMemcpyHostToDevice, P.stream));
    const long long blocks = std::min<long long>((rows + 255) / 256, (long long)P.sm_count * 8);
    bitstring_weights_kernel<RHO><<<(unsigned)std::max<long long>(blocks, 1), 256, 0, P.stream>>>(
        src, d_w.get(), D, rows, n, P.dim, one_digit, off);
    CUDA_CHECK(cudaGetLastError());
    size_t tmp_bytes = 0;
    CUDA_CHECK(cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, d_w.get(), d_w.get(), (int)M, P.stream));
    DevBuf<char> d_tmp(P, tmp_bytes);
    CUDA_CHECK(cub::DeviceScan::InclusiveSum(d_tmp.get(), tmp_bytes, d_w.get(), d_w.get(), (int)M, P.stream));
    search_sorted_kernel<<<(n_shots + 255) / 256, 256, 0, P.stream>>>(d_w.get(), M, d_u.get(), d_idx.get(), n_shots);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(out, d_idx.get(), sizeof(long long) * (size_t)n_shots, cudaMemcpyDeviceToHost, P.stream));
    CUDA_CHECK(cudaStreamSynchronize(P.stream));
}

#define PB200_TRY try {
#define PB200_CATCH                                         \
    }                                                       \
    catch (const Error& e) {                                \
        g_last_error = e.what();                            \
        return e.code;                                      \
    }                                                       \
    catch (const std::exception& e) {                       \
        g_last_error = e.what();                            \
        return PB200_ERR_INVALID;                           \
    }                                                       \
    return PB200_OK;

extern "C" {

int pb200_version(void) { return 100; }

const char* pb200_last_error(void) { return g_last_error.c_str(); }

int pb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

// checks of a plan description that need no device
static void check_desc(const pb200_plan_desc* d) {
    if (d->n_qudits < 1 || d->n_qudits > PB200_MAX_QUDITS) fail(PB200_ERR_INVALID, "n_qudits out of range");
    if (d->dim < 2 || d->dim > 4) fail(PB200_ERR_INVALID, "dim must be 2, 3 or 4");
    if (d->n_times < 2 || !d->sampling_times) fail(PB200_ERR_INVALID, "need >= 2 sampling times");
    if (d->n_drives < 0 || d->n_drives > PB200_MAX_DRIVES) fail(PB200_ERR_INVALID, "n_drives out of range");
    if (d->n_traj < 1) fail(PB200_ERR_INVALID, "n_traj must be >= 1");
    if (d->interp_order != 0 && d->interp_order != 1 && d->interp_order != 3)
        fail(PB200_ERR_INVALID, "interp_order must be 0, 1 or 3");
    for (int i = 1; i < d->n_times; ++i)
        if (!(d->sampling_times[i] > d->sampling_times[i - 1])) fail(PB200_ERR_INVALID, "sampling_times must increase");
    for (int q = 0; q < d->n_drives; ++q) {
        const pb200_drive_desc& dd = d->drives[q];
        if (dd.state_to < 0 || dd.state_to >= d->dim || dd.state_from < 0 || dd.state_from >= d->dim ||
            dd.state_to == dd.state_from)
            fail(PB200_ERR_INVALID, "drive %d: bad eigenstate indices", q);
    }
}

// shard_bits = 0: a whole state; else the plan holds shard `shard` of 2^shard_bits (checked by the caller)
static void create_plan(pb200_plan** out, const pb200_plan_desc* d, int shard_bits, int shard) {
    double Dd = std::pow((double)d->dim, d->n_qudits) / (double)(1LL << shard_bits);
    if (Dd * d->n_traj > 4.0e9) fail(PB200_ERR_UNSUPPORTED, "state too large: %g amplitudes", Dd * d->n_traj);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        fail(PB200_ERR_CUDA, "no CUDA device available: the pulser_b200 hot path has no CPU fallback");
    }
    if (d->device < 0 || d->device >= ndev) fail(PB200_ERR_INVALID, "device ordinal %d out of range", d->device);
    CUDA_CHECK(cudaSetDevice(d->device));
    std::unique_ptr<pb200_plan> h(new pb200_plan());
    Plan& P = h->p;
    P.desc = *d;
    P.times.assign(d->sampling_times, d->sampling_times + d->n_times);
    P.desc.sampling_times = nullptr;
    P.n = d->n_qudits; P.dim = d->dim; P.B = d->n_traj; P.n_drives = d->n_drives;
    long long D = 1;
    for (int i = 0; i < P.n; ++i) D *= P.dim;
    D >>= shard_bits;
    P.D = D;
    P.shard_bits = shard_bits; P.shard = shard;
    P.sm_count = device_setup(d->device);
    CUDA_CHECK(cudaStreamCreateWithFlags(&P.owned_stream.s, cudaStreamNonBlocking));
    P.stream = P.owned_stream.s;
    for (int i = 0; i < 3; ++i) P.buf[i].reset(P, (size_t)D * P.B);
    P.d_scratch.reset(P, 4096);
    P.tabs.assign(P.B, std::vector<DriveTables>(P.n_drives));
    P.tabs_set.assign(P.B, std::vector<bool>(P.n_drives, false));
    P.has_interaction = false;
    *out = h.release();
}

int pb200_plan_create(pb200_plan** out, const pb200_plan_desc* d) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_plan_create");
    if (!out || !d) fail(PB200_ERR_INVALID, "null argument");
    *out = nullptr;
    check_desc(d);
    create_plan(out, d, 0, 0);
    PB200_CATCH
}

int pb200_plan_create_shard(pb200_plan** out, const pb200_plan_desc* d, int32_t shard_bits, int32_t shard_index) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_plan_create_shard");
    if (!out || !d) fail(PB200_ERR_INVALID, "null argument");
    *out = nullptr;
    check_desc(d);
    if (shard_bits < 1 || shard_bits > PB200_MAX_SHARD_BITS)
        fail(PB200_ERR_INVALID, "shard_bits = %d: must be 1, 2 or 3 (2, 4 or 8 shards)", shard_bits);
    if (shard_index < 0 || shard_index >= (1 << shard_bits))
        fail(PB200_ERR_INVALID, "shard_index = %d out of range [0, %d)", shard_index, 1 << shard_bits);
    const int L = d->n_qudits - shard_bits;
    if (L < kTaylorTileBits || L > kShardMaxLocalBits)
        fail(PB200_ERR_INVALID, "N - shard_bits = %d: a shard holds 2^%d to 2^%d amplitudes", L, kTaylorTileBits,
             kShardMaxLocalBits);
    if (d->dim != 2 || d->n_drives != 1 || d->n_traj != 1)
        fail(PB200_ERR_UNSUPPORTED, "shards hold one state (n_traj = 1) of a d = 2 register with one drive (got d = %d, %d drives, "
                                    "%d trajectories)", d->dim, d->n_drives, d->n_traj);
    create_plan(out, d, shard_bits, shard_index);
    PB200_CATCH
}

int pb200_plan_destroy(pb200_plan* h) {
    if (!h) return PB200_OK;
    Plan& P = h->p;
    for (Plan* m : P.group)   // the other shards of a linked group are unlinked
        if (m != &P) m->group.clear();
    cudaSetDevice(P.desc.device);
    if (P.stream) cudaStreamSynchronize(P.stream);  // once: every buffer then returns to the pool without waiting
    delete h;
    return PB200_OK;
}

int pb200_plan_set_stream(pb200_plan* h, void* s) {
    PB200_TRY
    if (!h) fail(PB200_ERR_INVALID, "null plan");
    Plan& P = h->p;
    if (s) {
        P.owned_stream.reset();
        P.stream = (cudaStream_t)s;
    }
    PB200_CATCH
}

int pb200_plan_set_interaction(pb200_plan* h, int32_t traj0, int32_t count, const double* U, const uint8_t* bad,
                               int32_t shared) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_plan_set_interaction");
    if (!h || !U) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    if (P.desc.rydberg_state < 0) fail(PB200_ERR_INVALID, "plan has no interaction term (rydberg_state < 0)");
    if (shared && (count != 1 || traj0 != 0)) fail(PB200_ERR_INVALID, "shared interaction: traj0 = 0, count = 1");
    if (!shared) check_traj_range(P, traj0, count, "pb200_plan_set_interaction");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    const int N = P.n;
    const bool want_shared = shared != 0;
    if (!P.dint || P.dint_shared != want_shared) {
        P.dint.reset(P, (size_t)P.D * (want_shared ? 1 : P.B));
        P.cpl.reset(P, (size_t)N * N * (want_shared ? 1 : P.B));
        if (!want_shared) {
            CUDA_CHECK(cudaMemsetAsync(P.dint.get(), 0, sizeof(double) * (size_t)P.D * P.B, P.stream));
            CUDA_CHECK(cudaMemsetAsync(P.cpl.get(), 0, sizeof(double) * (size_t)N * N * P.B, P.stream));
        }
    }
    P.dint_shared = want_shared;
    P.dmin_traj.resize(want_shared ? 1 : P.B, 0.0);
    P.dmax_traj.resize(want_shared ? 1 : P.B, 0.0);
    if (P.has_slm) {
        P.dint2.reset(P, (size_t)P.D * (want_shared ? 1 : P.B));
        CUDA_CHECK(cudaMemsetAsync(P.dint2.get(), 0, sizeof(double) * (size_t)P.D * (want_shared ? 1 : P.B), P.stream));
        P.dmin2_traj.assign(want_shared ? 1 : P.B, 0.0);
        P.dmax2_traj.assign(want_shared ? 1 : P.B, 0.0);
    }
    DevBuf<double> dU2(P, (size_t)N * N);   // part 1; part 0 stays on the device in P.cpl
    std::vector<double> Uc((size_t)N * N);
    // part 0: pairs weighted by w (all pairs, or the pairs not touching the SLM mask); part 1: the pairs touching it
    for (int c = 0; c < count; ++c)
      for (int part = 0; part < (P.has_slm ? 2 : 1); ++part) {
        const double* Ui = U + (size_t)c * N * N;
        const uint8_t* bi = bad ? bad + (size_t)c * N : nullptr;
        for (int i = 0; i < N; ++i)
            for (int j = 0; j < N; ++j) {
                double u = (i < j) ? Ui[i * N + j] : (i > j ? Ui[j * N + i] : 0.0);
                if (bi && (bi[i] || bi[j])) u = 0.0;
                if (P.has_slm) {
                    const bool touched = ((P.slm_bits >> i) | (P.slm_bits >> j)) & 1ULL;
                    if (touched != (part == 1)) u = 0.0;
                }
                Uc[(size_t)i * N + j] = u;
            }
        double* dU = part == 0 ? P.cpl.get() + (want_shared ? 0 : (size_t)(traj0 + c) * N * N) : dU2.get();
        CUDA_CHECK(cudaMemcpyAsync(dU, Uc.data(), sizeof(double) * N * N, cudaMemcpyHostToDevice, P.stream));
        double* dst = (part == 0 ? P.dint : P.dint2).get() + (want_shared ? 0 : (size_t)(traj0 + c) * P.D);
        const int threads = 256;
        const long long blocks = std::min<long long>((P.D + threads - 1) / threads, (long long)P.sm_count * 16);
        dint_kernel<<<(unsigned)std::max<long long>(blocks, 1), threads, sizeof(double) * N * N, P.stream>>>(
            dst, dU, N, P.dim, P.desc.rydberg_state, P.D, P.shard_offset());
        CUDA_CHECK(cudaGetLastError());
        // bounds per |r>-count
        std::vector<double> mins(N + 1, 1e300), maxs(N + 1, -1e300);
        double* d_mins = P.d_scratch.get();
        double* d_maxs = d_mins + 64;
        CUDA_CHECK(cudaMemcpyAsync(d_mins, mins.data(), sizeof(double) * (N + 1), cudaMemcpyHostToDevice, P.stream));
        CUDA_CHECK(cudaMemcpyAsync(d_maxs, maxs.data(), sizeof(double) * (N + 1), cudaMemcpyHostToDevice, P.stream));
        dint_bounds_kernel<<<(unsigned)std::max<long long>(blocks, 1), threads, 0, P.stream>>>(
            dst, N, P.dim, P.desc.rydberg_state, P.D, d_mins, d_maxs, P.shard_offset());
        CUDA_CHECK(cudaGetLastError());
        CUDA_CHECK(cudaMemcpyAsync(mins.data(), d_mins, sizeof(double) * (N + 1), cudaMemcpyDeviceToHost, P.stream));
        CUDA_CHECK(cudaMemcpyAsync(maxs.data(), d_maxs, sizeof(double) * (N + 1), cudaMemcpyDeviceToHost, P.stream));
        CUDA_CHECK(cudaStreamSynchronize(P.stream));
        double mn = 1e300, mx = -1e300;
        for (int k = 0; k <= N; ++k)
            if (mins[k] <= maxs[k]) { mn = std::min(mn, mins[k]); mx = std::max(mx, maxs[k]); }
        const int slot = want_shared ? 0 : traj0 + c;
        if (part == 0) {
            P.dmin_traj[slot] = mn; P.dmax_traj[slot] = mx;
            if (want_shared) { P.dmin_cnt = mins; P.dmax_cnt = maxs; }
        } else {
            P.dmin2_traj[slot] = mn; P.dmax2_traj[slot] = mx;
        }
      }
    P.has_interaction = true;
    P.tay.w_knot.clear();
    PB200_CATCH
}

int pb200_plan_set_xy(pb200_plan* h, int32_t traj0, int32_t count, const double* Uxy, const uint8_t* bad, int32_t shared,
                      int32_t digit_u, int32_t digit_d) {
    PB200_TRY
    if (!h || !Uxy) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    if (shared && (count != 1 || traj0 != 0)) fail(PB200_ERR_INVALID, "shared couplings: traj0 = 0, count = 1");
    if (!shared) check_traj_range(P, traj0, count, "pb200_plan_set_xy");
    if (digit_u < 0 || digit_u >= P.dim || digit_d < 0 || digit_d >= P.dim || digit_u == digit_d)
        fail(PB200_ERR_INVALID, "bad eigenstate digits");
    if (P.n > 40) fail(PB200_ERR_UNSUPPORTED, "XY mode: at most 40 qudits");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    const int N = P.n;
    const bool want_shared = shared != 0;
    if (!P.d_xy || P.xy_shared != want_shared) {
        P.d_xy.reset(P, (size_t)N * N * (want_shared ? 1 : P.B));
        CUDA_CHECK(cudaMemsetAsync(P.d_xy.get(), 0, sizeof(double) * (size_t)N * N * (want_shared ? 1 : P.B), P.stream));
    }
    P.xy_shared = want_shared;
    P.xy_norm.resize(want_shared ? 1 : P.B, 0.0);
    P.xy_norm2.resize(want_shared ? 1 : P.B, 0.0);
    std::vector<double> Uc((size_t)N * N);
    for (int c = 0; c < count; ++c) {
        const double* Ui = Uxy + (size_t)c * N * N;
        const uint8_t* bi = bad ? bad + (size_t)c * N : nullptr;
        double nrm = 0.0, nrm2 = 0.0;
        for (int i = 0; i < N; ++i)
            for (int j = 0; j < N; ++j) {
                double u = (i < j) ? Ui[i * N + j] : (i > j ? Ui[j * N + i] : 0.0);
                if (bi && (bi[i] || bi[j])) u = 0.0;
                Uc[(size_t)i * N + j] = u;
                const bool touched = P.has_slm && (((P.slm_bits >> i) | (P.slm_bits >> j)) & 1ULL);
                if (i < j) { if (touched) nrm2 += std::fabs(u); else nrm += std::fabs(u); }
            }
        const int slot = want_shared ? 0 : traj0 + c;
        CUDA_CHECK(cudaMemcpyAsync(P.d_xy.get() + (size_t)slot * N * N, Uc.data(), sizeof(double) * N * N, cudaMemcpyHostToDevice, P.stream));
        CUDA_CHECK(cudaStreamSynchronize(P.stream));
        P.xy_norm[slot] = nrm; P.xy_norm2[slot] = nrm2;
    }
    P.xy_u = digit_u; P.xy_d = digit_d;
    P.has_xy = true;
    PB200_CATCH
}

int pb200_plan_set_slm_mask(pb200_plan* h, const uint8_t* masked, const double* coeff) {
    PB200_TRY
    if (!h || !masked || !coeff) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    if (P.has_interaction || P.has_xy)
        fail(PB200_ERR_STATE, "pb200_plan_set_slm_mask must precede pb200_plan_set_interaction / pb200_plan_set_xy");
    if (P.n > 63) fail(PB200_ERR_UNSUPPORTED, "SLM mask: at most 63 qudits");
    const int nt = (int)P.times.size();
    for (int i = 0; i < nt; ++i)
        if (!std::isfinite(coeff[i])) fail(PB200_ERR_INVALID, "non-finite SLM coefficient sample");
    P.slm_bits = 0;
    for (int k = 0; k < P.n; ++k)
        if (masked[k]) P.slm_bits |= 1ULL << k;
    P.slm_coef = make_interpolant<double>(P.times.data(), coeff, nt, P.desc.interp_order);
    P.has_slm = P.slm_bits != 0;
    P.fine_cache.valid = false;   // the 0 -> 1 switch of the mask is a jump interval
    PB200_CATCH
}

int pb200_plan_set_drive(pb200_plan* h, int32_t drive, int32_t traj0, int32_t count, const double* coef,
                         const double* det) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_plan_set_drive");
    if (!h || !coef || !det) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    if (drive < 0 || drive >= P.n_drives) fail(PB200_ERR_INVALID, "drive index out of range");
    check_traj_range(P, traj0, count, "pb200_plan_set_drive");
    const int rows = P.desc.drives[drive].uniform ? 1 : P.n;
    const int nt = (int)P.times.size();
    for (int c = 0; c < count; ++c) {
        DriveTables& T = P.tabs[traj0 + c][drive];
        T.coef.resize(rows); T.det.resize(rows);
        T.coef_scale.assign(rows, 0.0); T.det_scale.assign(rows, 0.0);
        for (int r = 0; r < rows; ++r) {
            const cplx* y = reinterpret_cast<const cplx*>(coef) + ((size_t)c * rows + r) * nt;
            const double* dd = det + ((size_t)c * rows + r) * nt;
            T.coef[r] = make_interpolant<cplx>(P.times.data(), y, nt, P.desc.interp_order);
            T.det[r] = make_interpolant<double>(P.times.data(), dd, nt, P.desc.interp_order);
            for (int i = 0; i < nt; ++i) {
                if (!std::isfinite(y[i].real()) || !std::isfinite(y[i].imag()) || !std::isfinite(dd[i]))
                    fail(PB200_ERR_INVALID, "non-finite sample in drive table");
                T.coef_scale[r] = std::max(T.coef_scale[r], std::abs(y[i]));
                T.det_scale[r] = std::max(T.det_scale[r], std::fabs(dd[i]));
            }
        }
        P.tabs_set[traj0 + c][drive] = true;
        P.fine_cache.valid = false; P.ctrl_Kc = -1.0; P.tay.valid = false; P.tay.w_knot.clear();
    }
    PB200_CATCH
}

int pb200_plan_set_dissipator(pb200_plan* h, int32_t n_pairs, const double* generators) {
    PB200_TRY
    if (!h || !generators) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    if (P.dim > 3) fail(PB200_ERR_UNSUPPORTED, "dissipator: d <= 3 only");
    if (n_pairs < 1 || 2 * n_pairs != P.n) fail(PB200_ERR_INVALID, "dissipator: the plan must hold 2*n_pairs qudits");
    const int dd = P.dim * P.dim;
    P.diss_gen.assign(n_pairs, std::vector<cplx>((size_t)dd * dd));
    const cplx* src = reinterpret_cast<const cplx*>(generators);
    for (int k = 0; k < n_pairs; ++k)
        for (int i = 0; i < dd * dd; ++i) {
            const cplx z = src[(size_t)k * dd * dd + i];
            if (!std::isfinite(z.real()) || !std::isfinite(z.imag())) fail(PB200_ERR_INVALID, "non-finite generator");
            P.diss_gen[k][i] = z;
        }
    P.has_diss = true;
    P.diss_tay = diss_taylor_analyse(P.diss_gen, P.dim);
    P.tay.valid = false;
    PB200_CATCH
}

int pb200_plan_set_collapse(pb200_plan* h, int32_t n_ops, const double* ops, uint64_t seed) {
    PB200_TRY
    if (!h || !ops || n_ops < 1) fail(PB200_ERR_INVALID, "bad argument");
    Plan& P = h->p;
    if (P.has_diss) fail(PB200_ERR_STATE, "plan already carries a dissipator (density-matrix mode)");
    const int d = P.dim;
    P.jump_ops.assign(n_ops, std::vector<cplx>((size_t)d * d));
    P.jump_ldl.assign(n_ops, std::vector<double>(d, 0.0));
    P.jump_ldl_full.assign(n_ops, std::vector<cplx>((size_t)d * d, cplx(0)));
    P.jump_diag = true;
    const cplx* src = reinterpret_cast<const cplx*>(ops);
    for (int op = 0; op < n_ops; ++op) {
        for (int q = 0; q < d * d; ++q) P.jump_ops[op][q] = src[(size_t)op * d * d + q];
        for (int a = 0; a < d; ++a)
            for (int b = 0; b < d; ++b) {
                cplx acc = 0.0;  // (L^+ L)[a][b] = sum_c conj(L[c][a]) L[c][b]
                for (int c = 0; c < d; ++c) acc += std::conj(P.jump_ops[op][c * d + a]) * P.jump_ops[op][c * d + b];
                if (a == b) P.jump_ldl[op][a] = acc.real();
                else if (std::abs(acc) > 1e-12) P.jump_diag = false;
                P.jump_ldl_full[op][a * d + b] = acc;
            }
    }
    P.rng.seed(seed);
    std::uniform_real_distribution<double> uni(0.0, 1.0);
    P.thresholds.resize(P.B);
    for (double& r : P.thresholds) r = uni(P.rng);
    P.jump_count.assign(P.B, 0);
    P.has_collapse = true;
    PB200_CATCH
}

int pb200_plan_jump_counts(pb200_plan* h, int64_t* jumps) {
    PB200_TRY
    if (!h || !jumps) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    for (int i = 0; i < P.B; ++i) jumps[i] = P.has_collapse ? (int64_t)P.jump_count[i] : 0;
    PB200_CATCH
}

int pb200_state_set(pb200_plan* h, int32_t traj0, int32_t count, const double* psi, int64_t basis_index,
                    int32_t broadcast) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_state_set");
    if (!h) fail(PB200_ERR_INVALID, "null plan");
    Plan& P = h->p;
    check_traj_range(P, traj0, count, "pb200_state_set");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    c2* cur = P.buf[P.cur].get();
    for (int c = 0; c < count; ++c) {
        c2* dst = cur + (size_t)(traj0 + c) * P.D;
        if (psi) {
            const double* src = broadcast ? psi : psi + (size_t)c * P.D * 2;
            CUDA_CHECK(cudaMemcpyAsync(dst, src, sizeof(c2) * (size_t)P.D, cudaMemcpyHostToDevice, P.stream));
        } else {
            // a shard takes the global index: the shard that owns it sets it, the others zero their slice
            if (basis_index < 0 || basis_index >= (P.D << P.shard_bits)) fail(PB200_ERR_INVALID, "basis_index out of range");
            long long local = basis_index - P.shard_offset();
            if (local >= P.D) local = -1;
            const long long blocks = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 16);
            set_basis_kernel<<<(unsigned)blocks, 256, 0, P.stream>>>(dst, P.D, local);
            CUDA_CHECK(cudaGetLastError());
        }
    }
    CUDA_CHECK(cudaStreamSynchronize(P.stream));
    P.state_set = true;
    PB200_CATCH
}

int pb200_state_get(pb200_plan* h, int32_t traj0, int32_t count, double* psi) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_state_get");
    if (!h || !psi) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    check_traj_range(P, traj0, count, "pb200_state_get");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    CUDA_CHECK(cudaMemcpyAsync(psi, P.buf[P.cur].get() + (size_t)traj0 * P.D, sizeof(c2) * (size_t)P.D * count,
                               cudaMemcpyDeviceToHost, P.stream));
    CUDA_CHECK(cudaStreamSynchronize(P.stream));
    PB200_CATCH
}

int pb200_state_probabilities(pb200_plan* h, int32_t traj0, int32_t count, double* probs) {
    PB200_TRY
    if (!h || !probs) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    check_traj_range(P, traj0, count, "pb200_state_probabilities");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    // reuse a scratch state buffer for the doubles
    double* tmp = reinterpret_cast<double*>(P.buf[(P.cur + 1) % 3].get());
    const long long total = P.D * count;
    const long long blocks = std::min<long long>((total + 255) / 256, (long long)P.sm_count * 16);
    prob_kernel<<<(unsigned)blocks, 256, 0, P.stream>>>(P.buf[P.cur].get() + (size_t)traj0 * P.D, tmp, total);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(probs, tmp, sizeof(double) * (size_t)total, cudaMemcpyDeviceToHost, P.stream));
    CUDA_CHECK(cudaStreamSynchronize(P.stream));
    PB200_CATCH
}

int pb200_state_norm2(pb200_plan* h, int32_t traj0, int32_t count, double* norms2) {
    PB200_TRY
    if (!h || !norms2) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    check_traj_range(P, traj0, count, "pb200_state_norm2");
    if (count > 4096) fail(PB200_ERR_INVALID, "pb200_state_norm2: trajectory range: at most 4096 per call");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    const long long blocks = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 4);
    dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)count);
    device_sum(P, P.d_scratch.get(), count, norms2, [&] {
        norm2_kernel<<<grid, 256, 0, P.stream>>>(P.buf[P.cur].get() + (size_t)traj0 * P.D, P.D, P.d_scratch.get());
    });
    PB200_CATCH
}

int pb200_state_occupation(pb200_plan* h, int32_t traj0, int32_t count, int32_t digit, double* occ) {
    PB200_TRY
    if (!h || !occ) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    check_traj_range(P, traj0, count, "pb200_state_occupation");
    if (digit < 0 || digit >= P.dim) fail(PB200_ERR_INVALID, "digit out of range");
    reduce_occupation<false>(P, P.buf[P.cur].get() + (size_t)traj0 * P.D, P.D, P.D, P.shard_offset(), P.n, count, digit,
                             occ);
    PB200_CATCH
}

int pb200_state_correlation(pb200_plan* h, int32_t traj0, int32_t count, int32_t digit, double* corr) {
    PB200_TRY
    if (!h || !corr) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    check_traj_range(P, traj0, count, "pb200_state_correlation");
    if (digit < 0 || digit >= P.dim) fail(PB200_ERR_INVALID, "digit out of range");
    if (P.n > 40) fail(PB200_ERR_UNSUPPORTED, "too many qudits for the correlation matrix");
    reduce_correlation<false>(P, P.buf[P.cur].get() + (size_t)traj0 * P.D, P.D, P.D, P.shard_offset(), P.n, count, digit,
                              corr);
    PB200_CATCH
}

int pb200_state_energy(pb200_plan* h, double t_us, double* energy, double* h2) {
    PB200_TRY
    if (!h || !energy || !h2) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    refuse_shard(P, "pb200_state_energy", "pb200_shards_energy");
    check_drives_set(P, "pb200_state_energy");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    c2* psi = P.buf[P.cur].get();
    c2* hpsi = P.buf[(P.cur + 2) % 3].get();
    long long launches = 0;
    apply_h_device(P, t_us, psi, hpsi, launches);
    DevBuf<double> d_acc(P, 2 * (size_t)P.B);
    const long long blocks = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 8);
    dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)P.B);
    std::vector<double> acc(2 * (size_t)P.B);
    device_sum(P, d_acc.get(), acc.size(), acc.data(), [&] {
        dot2_kernel<<<grid, 256, 0, P.stream>>>(psi, hpsi, P.D, d_acc.get());  // Re<psi, H psi>, <H psi, H psi>
    });
    for (int b = 0; b < P.B; ++b) { energy[b] = acc[2 * b]; h2[b] = acc[2 * b + 1]; }
    PB200_CATCH
}

int pb200_state_overlap(pb200_plan* h, int32_t traj0, int32_t count, const double* phi, double* out) {
    PB200_TRY
    if (!h || !phi || !out) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    check_traj_range(P, traj0, count, "pb200_state_overlap");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    c2* d_phi = P.buf[(P.cur + 1) % 3].get();
    CUDA_CHECK(cudaMemcpyAsync(d_phi, phi, sizeof(c2) * (size_t)P.D, cudaMemcpyHostToDevice, P.stream));
    DevBuf<double> d_acc(P, 2 * (size_t)count);
    const long long blocks = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 8);
    dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)count);
    device_sum(P, d_acc.get(), d_acc.size(), out, [&] {
        overlap_kernel<<<grid, 256, 0, P.stream>>>(d_phi, P.buf[P.cur].get() + (size_t)traj0 * P.D, P.D, d_acc.get());
    });
    PB200_CATCH
}

int pb200_state_expect(pb200_plan* h, int32_t traj0, int32_t count, const pb200_op_terms* op, double* out) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_state_expect");
    if (!h || !out) fail(PB200_ERR_INVALID, "pb200_state_expect: null argument");
    Plan& P = h->p;
    refuse_shard(P, "pb200_state_expect", "pb200_shards_expect");
    if (P.has_diss)
        fail(PB200_ERR_UNSUPPORTED, "pb200_state_expect: the plan holds a vectorised density matrix, not state vectors");
    check_traj_range(P, traj0, count, "pb200_state_expect");
    check_op_terms(op, P.n, P.dim, "pb200_state_expect");
    if (!P.state_set) fail(PB200_ERR_STATE, "pb200_state_expect: no state set");
    std::fill(out, out + 2 * (size_t)count, 0.0);
    const ExpHost H = exp_host(op, P.n, P.dim, P.n);
    if (H.n_chunks == 0) return PB200_OK;
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    const DevBuf<char> X = upload_exp(H, P);
    DevBuf<double> d_acc(P, 2 * (size_t)count);
    const c2* psi = P.buf[P.cur].get() + (size_t)traj0 * P.D;
    ExpSrc src{};
    src.p[0] = psi; src.shard = 0; src.local_bits = P.n;
    device_sum(P, d_acc.get(), d_acc.size(), out, [&] { launch_expect<false>(P, P.D, H, X.get(), src, psi, count, d_acc.get()); });
    PB200_CATCH
}

int pb200_state_sample(pb200_plan* h, int32_t traj, int32_t one_digit, const double* uniforms, int32_t n_shots,
                       int64_t* out) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_state_sample");
    if (!h || !uniforms || !out || n_shots < 1) fail(PB200_ERR_INVALID, "bad argument");
    Plan& P = h->p;
    if (traj < 0 || traj >= P.B) fail(PB200_ERR_INVALID, "trajectory out of range");
    if (one_digit < 0 || one_digit >= P.dim) fail(PB200_ERR_INVALID, "one_digit out of range");
    // a shard samples its own slice: M = its 2^L bitstrings, out[i] = the low L bits of the global bitstring
    sample_bitstrings<false>(P, P.buf[P.cur].get() + (size_t)traj * P.D, P.D, P.D, P.shard_offset(), P.n, P.n - P.shard_bits,
                             one_digit, uniforms, n_shots, out);
    PB200_CATCH
}

int pb200_state_copy(pb200_plan* dst, int32_t dst_traj, pb200_plan* src, int32_t src_traj) {
    PB200_TRY
    if (!dst || !src) fail(PB200_ERR_INVALID, "null argument");
    Plan& A = dst->p;
    Plan& S = src->p;
    if (A.shard_bits || S.shard_bits) fail(PB200_ERR_UNSUPPORTED, "pb200_state_copy: shards hold a slice of a state, not a state");
    if (!S.state_set) fail(PB200_ERR_STATE, "pb200_state_copy: the source plan has no state");
    if (A.D != S.D || A.dim != S.dim) fail(PB200_ERR_INVALID, "pb200_state_copy: different Hilbert spaces");
    if (A.desc.device != S.desc.device) fail(PB200_ERR_UNSUPPORTED, "pb200_state_copy: plans on different devices");
    if (dst_traj < 0 || dst_traj >= A.B || src_traj < 0 || src_traj >= S.B) fail(PB200_ERR_INVALID, "trajectory range");
    if (A.B > 1 && !A.state_set) fail(PB200_ERR_STATE, "pb200_state_copy: set the other trajectories of the destination first");
    CUDA_CHECK(cudaSetDevice(A.desc.device));
    CUDA_CHECK(cudaStreamSynchronize(S.stream));  // the source state is complete
    CUDA_CHECK(cudaMemcpyAsync(A.buf[A.cur].get() + (size_t)dst_traj * A.D, S.buf[S.cur].get() + (size_t)src_traj * S.D,
                               sizeof(c2) * (size_t)A.D, cudaMemcpyDeviceToDevice, A.stream));
    CUDA_CHECK(cudaStreamSynchronize(A.stream));
    A.state_set = true;
    PB200_CATCH
}

int pb200_state_device_ptr(pb200_plan* h, void** dptr) {
    PB200_TRY
    if (!h || !dptr) fail(PB200_ERR_INVALID, "null argument");
    *dptr = h->p.buf[h->p.cur].get();
    PB200_CATCH
}

// ---- reductions of density matrices (plans with a dissipator) ------------------------------------------------------
// The plan holds vec(rho) of N = n / 2 physical qudits: D = dim^N, trajectory b at buf + b D^2.  A shard of vec(rho)
// (one trajectory) holds the rows [r0, r0 + rows) of rho, rows = D / 2^shard_bits: each reduction returns the share of
// those rows, which the caller sums over the shards (the kernels never read a peer's rows).
struct DensityGeom { int n; long long D, rows, r0; };

static DensityGeom density_geom(const Plan& P, const char* who) {
    if (!P.has_diss)
        fail(PB200_ERR_UNSUPPORTED, "%s: the plan holds state vectors, not a density matrix (no dissipator)", who);
    if (!P.state_set) fail(PB200_ERR_STATE, "%s: no state set", who);
    DensityGeom G{P.n / 2, 1, 0, 0};
    for (int k = 0; k < G.n; ++k) G.D *= P.dim;
    G.rows = G.D >> P.shard_bits;
    G.r0 = (long long)P.shard * G.rows;
    return G;
}

static const c2* density_at(const Plan& P, const DensityGeom& G, int traj) {
    return P.buf[P.cur].get() + (size_t)traj * G.rows * G.D;
}

int pb200_density_trace(pb200_plan* h, int32_t traj0, int32_t count, double* trace) {
    PB200_TRY
    if (!h || !trace) fail(PB200_ERR_INVALID, "pb200_density_trace: null argument");
    Plan& P = h->p;
    const DensityGeom G = density_geom(P, "pb200_density_trace");
    check_traj_range(P, traj0, count, "pb200_density_trace");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    DevBuf<double> d_acc(P, 2 * (size_t)count);
    std::vector<double> acc(2 * (size_t)count);
    const long long blocks = std::min<long long>((G.rows + 255) / 256, (long long)P.sm_count * 4);
    dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)count);
    device_sum(P, d_acc.get(), acc.size(), acc.data(), [&] {
        density_trace_kernel<<<grid, 256, 0, P.stream>>>(density_at(P, G, traj0) + G.r0, G.D, G.rows, d_acc.get());
    });
    for (int c = 0; c < count; ++c) trace[c] = acc[2 * (size_t)c];
    PB200_CATCH
}

int pb200_density_occupation(pb200_plan* h, int32_t traj0, int32_t count, int32_t digit, double* occ) {
    PB200_TRY
    if (!h || !occ) fail(PB200_ERR_INVALID, "pb200_density_occupation: null argument");
    Plan& P = h->p;
    const DensityGeom G = density_geom(P, "pb200_density_occupation");
    check_traj_range(P, traj0, count, "pb200_density_occupation");
    if (digit < 0 || digit >= P.dim) fail(PB200_ERR_INVALID, "pb200_density_occupation: digit out of range");
    reduce_occupation<true>(P, density_at(P, G, traj0) + G.r0, G.D, G.rows, G.r0, G.n, count, digit, occ);
    PB200_CATCH
}

int pb200_density_correlation(pb200_plan* h, int32_t traj0, int32_t count, int32_t digit, double* corr) {
    PB200_TRY
    if (!h || !corr) fail(PB200_ERR_INVALID, "pb200_density_correlation: null argument");
    Plan& P = h->p;
    const DensityGeom G = density_geom(P, "pb200_density_correlation");
    check_traj_range(P, traj0, count, "pb200_density_correlation");
    if (digit < 0 || digit >= P.dim) fail(PB200_ERR_INVALID, "pb200_density_correlation: digit out of range");
    reduce_correlation<true>(P, density_at(P, G, traj0) + G.r0, G.D, G.rows, G.r0, G.n, count, digit, corr);
    PB200_CATCH
}

int pb200_density_expect(pb200_plan* h, int32_t traj0, int32_t count, const pb200_op_terms* op, double* out) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_density_expect");
    if (!h || !out) fail(PB200_ERR_INVALID, "pb200_density_expect: null argument");
    Plan& P = h->p;
    const DensityGeom G = density_geom(P, "pb200_density_expect");
    check_traj_range(P, traj0, count, "pb200_density_expect");
    check_op_terms(op, G.n, P.dim, "pb200_density_expect");
    std::fill(out, out + 2 * (size_t)count, 0.0);
    const int local_bits = G.n - P.shard_bits;
    const ExpHost H = exp_host(op, G.n, P.dim, local_bits);
    if (H.n_chunks == 0) return PB200_OK;
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    const DevBuf<char> X = upload_exp(H, P);
    DevBuf<double> d_acc(P, 2 * (size_t)count);
    const c2* rho = density_at(P, G, traj0);
    ExpSrc src{};
    src.p[0] = rho; src.shard = 0; src.local_bits = local_bits;
    if (P.shard_bits) {   // the stored rows of a shard (d = 2): rows (shard << local_bits) | s of D entries
        src.p[P.shard] = rho; src.shard = P.shard; src.row_len = G.D;
    }
    device_sum(P, d_acc.get(), d_acc.size(), out,
               [&] { launch_expect<true>(P, G.rows, H, X.get(), src, rho, count, d_acc.get()); });
    PB200_CATCH
}

int pb200_density_energy(pb200_plan* h, pb200_plan* ham, double t_us, int32_t traj0, int32_t count, double* energy,
                         double* h2) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_density_energy");
    if (!h || !ham || !energy || !h2) fail(PB200_ERR_INVALID, "pb200_density_energy: null argument");
    Plan& P = h->p;
    const Plan& Q = ham->p;
    const DensityGeom G = density_geom(P, "pb200_density_energy");
    check_traj_range(P, traj0, count, "pb200_density_energy");
    if (P.has_xy || Q.has_xy)
        fail(PB200_ERR_UNSUPPORTED, "pb200_density_energy: XY registers (the exchange term is not evaluated)");
    if (Q.has_diss || Q.has_collapse || Q.shard_bits || Q.B != 1)
        fail(PB200_ERR_INVALID, "pb200_density_energy: the Hamiltonian plan must be a single-state plan without noise");
    if (Q.n != G.n || Q.dim != P.dim)
        fail(PB200_ERR_INVALID, "pb200_density_energy: the Hamiltonian plan has %d qudits of dimension %d, the density "
             "matrix %d of dimension %d", Q.n, Q.dim, G.n, P.dim);
    if (Q.desc.device != P.desc.device)
        fail(PB200_ERR_UNSUPPORTED, "pb200_density_energy: plans on different devices (a shard on device %d needs a "
             "Hamiltonian plan of its own there)", P.desc.device);
    if (G.n > kDensityMaxQudits) fail(PB200_ERR_UNSUPPORTED, "pb200_density_energy: at most %d qudits", kDensityMaxQudits);
    check_drives_set(Q, "pb200_density_energy");
    const ExpParams E = params_at(Q, t_us);
    DensityH dh{};
    dh.n = G.n; dh.dim = Q.dim; dh.n_drives = Q.n_drives;
    for (int q = 0; q < Q.n_drives; ++q) {
        dh.to[q] = Q.desc.drives[q].state_to;
        dh.from[q] = Q.desc.drives[q].state_from;
        for (int k = 0; k < G.n; ++k) {
            const cplx g = E.g[pidx(Q, 0, q, k)];
            dh.g[q][k] = {g.real(), g.imag()};
            dh.th[q][k] = E.th[pidx(Q, 0, q, k)];
        }
    }
    dh.dint = Q.has_interaction ? Q.dint.get() : nullptr;  // complete: pb200_plan_set_interaction synchronises
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    DevBuf<double> d_acc(P, 2 * (size_t)count);
    std::vector<double> acc(2 * (size_t)count);
    const long long blocks = (G.rows + 255) / 256;
    dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)count);
    device_sum(P, d_acc.get(), acc.size(), acc.data(), [&] {
        // a shard sums over the rows it stores (Tr(rho H), Tr(rho H^2)): (H rho)[a, r] would read the rows of its peers
        if (P.shard_bits)
            density_energy_rows_kernel<<<grid, 256, 0, P.stream>>>(density_at(P, G, traj0), G.D, G.rows, G.r0, dh,
                                                                   d_acc.get());
        else
            density_energy_kernel<<<grid, 256, 0, P.stream>>>(density_at(P, G, traj0), G.D, dh, d_acc.get());
    });
    for (int c = 0; c < count; ++c) { energy[c] = acc[2 * (size_t)c]; h2[c] = acc[2 * (size_t)c + 1]; }
    PB200_CATCH
}

int pb200_density_overlap(pb200_plan* h, int32_t traj0, int32_t count, const double* phi, double* out) {
    PB200_TRY
    if (!h || !phi || !out) fail(PB200_ERR_INVALID, "pb200_density_overlap: null argument");
    Plan& P = h->p;
    const DensityGeom G = density_geom(P, "pb200_density_overlap");
    check_traj_range(P, traj0, count, "pb200_density_overlap");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    c2* d_phi = P.buf[(P.cur + 1) % 3].get();  // scratch of B D^2 >= D amplitudes
    CUDA_CHECK(cudaMemcpyAsync(d_phi, phi, sizeof(c2) * (size_t)G.D, cudaMemcpyHostToDevice, P.stream));
    DevBuf<double> d_acc(P, 2 * (size_t)count);
    const long long blocks = std::min<long long>(G.rows, (long long)P.sm_count * 8);
    dim3 grid((unsigned)std::max<long long>(blocks, 1), (unsigned)count);
    device_sum(P, d_acc.get(), d_acc.size(), out, [&] {
        density_overlap_kernel<<<grid, 256, 0, P.stream>>>(d_phi, density_at(P, G, traj0), G.D, G.rows, G.r0, d_acc.get());
    });
    PB200_CATCH
}

int pb200_density_sample(pb200_plan* h, int32_t traj, int32_t one_digit, const double* uniforms, int32_t n_shots,
                         int64_t* out) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_density_sample");
    if (!h || !uniforms || !out || n_shots < 1) fail(PB200_ERR_INVALID, "pb200_density_sample: bad argument");
    Plan& P = h->p;
    const DensityGeom G = density_geom(P, "pb200_density_sample");
    if (traj < 0 || traj >= P.B) fail(PB200_ERR_INVALID, "pb200_density_sample: trajectory out of range");
    if (one_digit < 0 || one_digit >= P.dim) fail(PB200_ERR_INVALID, "pb200_density_sample: one_digit out of range");
    sample_bitstrings<true>(P, density_at(P, G, traj) + G.r0, G.D, G.rows, G.r0, G.n, G.n - P.shard_bits, one_digit,
                            uniforms, n_shots, out);
    PB200_CATCH
}

int pb200_propagate(pb200_plan* h, double t_start, double t_stop, const pb200_run_opts* opts, pb200_run_stats* stats) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_propagate");
    if (!h) fail(PB200_ERR_INVALID, "null plan");
    refuse_shard(h->p, "pb200_propagate", "pb200_shards_propagate");
    CUDA_CHECK(cudaSetDevice(h->p.desc.device));
    propagate(h->p, t_start, t_stop, opts, stats);
    PB200_CATCH
}

int pb200_apply_h(pb200_plan* h, int32_t traj, double t_us, const double* in, double* out) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_apply_h");
    if (!h || !in || !out) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    refuse_shard(P, "pb200_apply_h", "pb200_shards_apply_h");
    if (traj < 0 || traj >= P.B) fail(PB200_ERR_INVALID, "trajectory out of range");
    check_drives_set(P, "pb200_apply_h");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    c2* bin = P.buf[(P.cur + 1) % 3].get();
    c2* bout = P.buf[(P.cur + 2) % 3].get();
    // the kernels run over the whole batch: zero the other trajectories' input
    CUDA_CHECK(cudaMemsetAsync(bin, 0, sizeof(c2) * (size_t)P.D * P.B, P.stream));
    CUDA_CHECK(cudaMemcpyAsync(bin + (size_t)traj * P.D, in, sizeof(c2) * (size_t)P.D, cudaMemcpyHostToDevice, P.stream));
    long long launches = 0;
    apply_h_device(P, t_us, bin, bout, launches);
    CUDA_CHECK(cudaMemcpyAsync(out, bout + (size_t)traj * P.D, sizeof(c2) * (size_t)P.D, cudaMemcpyDeviceToHost, P.stream));
    CUDA_CHECK(cudaStreamSynchronize(P.stream));
    PB200_CATCH
}

int pb200_coefficients_at(pb200_plan* h, int32_t traj, int32_t drive, int32_t row, double t_us, double* out3) {
    PB200_TRY
    if (!h || !out3) fail(PB200_ERR_INVALID, "null argument");
    Plan& P = h->p;
    if (traj < 0 || traj >= P.B || drive < 0 || drive >= P.n_drives) fail(PB200_ERR_INVALID, "index out of range");
    if (!P.tabs_set[traj][drive]) fail(PB200_ERR_STATE, "drive not set");
    const DriveTables& T = P.tabs[traj][drive];
    if (row < 0 || row >= (int)T.coef.size()) fail(PB200_ERR_INVALID, "row out of range");
    const cplx c = eval_at(T.coef[row], P.times, t_us, P.desc.interp_order);
    out3[0] = c.real(); out3[1] = c.imag();
    out3[2] = eval_at(T.det[row], P.times, t_us, P.desc.interp_order);
    PB200_CATCH
}

int pb200_bench_apply(pb200_plan* h, double t_us, int32_t reps, double* ms_out, int64_t* launches_out) {
    PB200_TRY
    if (!h || !ms_out || reps < 1) fail(PB200_ERR_INVALID, "bad argument");
    Plan& P = h->p;
    refuse_shard(P, "pb200_bench_apply", "pb200_shards_apply_h");
    if (!P.state_set) fail(PB200_ERR_STATE, "no state set");
    CUDA_CHECK(cudaSetDevice(P.desc.device));
    c2* in = P.buf[P.cur].get();
    c2* outb = P.buf[(P.cur + 1) % 3].get();
    long long launches = 0;
    const ApplyH A = apply_h_device(P, t_us, in, outb, launches);  // warm-up + table upload
    CUDA_CHECK(cudaStreamSynchronize(P.stream));
    EventPair evs;
    launches = 0;
    evs.start(P.stream);
    for (int r = 0; r < reps; ++r) A.launch(P, in, outb, launches);
    *ms_out = evs.stop_ms(P.stream);
    CUDA_CHECK(cudaGetLastError());
    if (launches_out) *launches_out = launches;
    PB200_CATCH
}

int pb200_shards_link(pb200_plan** plans, int32_t count) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_shards_link");
    if (!plans) fail(PB200_ERR_INVALID, "null argument");
    if (count != 2 && count != 4 && count != 8) fail(PB200_ERR_INVALID, "pb200_shards_link: count = %d, must be 2, 4 or 8", count);
    std::vector<Plan*> G(count);
    for (int i = 0; i < count; ++i) {
        if (!plans[i]) fail(PB200_ERR_INVALID, "pb200_shards_link: null plan");
        G[i] = &plans[i]->p;
    }
    for (int i = 0; i < count; ++i) {
        Plan& P = *G[i];
        if ((1 << P.shard_bits) != count) fail(PB200_ERR_INVALID, "pb200_shards_link: plans[%d] is not one of %d shards", i, count);
        if (P.shard != i) fail(PB200_ERR_INVALID, "pb200_shards_link: plans[%d] is shard %d (plans[i] must be shard i)", i, P.shard);
        if (P.n != G[0]->n || P.times != G[0]->times || P.desc.interp_order != G[0]->desc.interp_order)
            fail(PB200_ERR_INVALID, "pb200_shards_link: the shards differ in N, sampling times or interpolation order");
        if (P.has_interaction != G[0]->has_interaction || (P.has_interaction && !P.dint_shared))
            fail(PB200_ERR_INVALID, "pb200_shards_link: every shard needs the same (shared) interaction");
        if (!P.tabs_set[0][0]) fail(PB200_ERR_STATE, "pb200_shards_link: the drive of shard %d is not set", i);
        // a master equation: every shard carries the same dissipator, so that each one's a-priori bound (w_knot, m_0)
        // and with it the group's schedule are those of the unsharded plan
        if (P.has_diss != G[0]->has_diss || P.diss_gen != G[0]->diss_gen)
            fail(PB200_ERR_INVALID, "pb200_shards_link: the shards carry different dissipators");
        if (!taylor_prepare(P)) fail(PB200_ERR_UNSUPPORTED, "pb200_shards_link: no Taylor propagator for this sequence: %s", g_taylor_why);
        // vec(rho) runs the batch gather, whose per-bit table holds the column drive -conj(omega)
        if (!P.tay.drive_uniform && !P.has_diss)
            fail(PB200_ERR_UNSUPPORTED, "pb200_shards_link: shards need one drive coefficient for every qubit (per-qubit drive "
                                        "amplitudes are not sharded; per-qubit detuning is)");
    }
    // peer access between distinct devices of neighbouring shards (a flip of one shard bit)
    for (int i = 0; i < count; ++i)
        for (int q = 0; (1 << q) < count; ++q) {
            const int di = G[i]->desc.device, dj = G[i ^ (1 << q)]->desc.device;
            if (di == dj) continue;
            int can = 0;
            CUDA_CHECK(cudaDeviceCanAccessPeer(&can, di, dj));
            if (!can) fail(PB200_ERR_UNSUPPORTED, "pb200_shards_link: device %d cannot access the memory of device %d (no peer access)", di, dj);
            CUDA_CHECK(cudaSetDevice(di));
            const cudaError_t e = cudaDeviceEnablePeerAccess(dj, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
            else CUDA_CHECK(e);
        }
    // spectral bounds of the whole interaction diagonal: min / max over the shards' slices, so that the host schedule
    // (taylor_bounds) is the one of the unsharded plan
    if (G[0]->has_interaction) {
        std::vector<double> mins = G[0]->dmin_cnt, maxs = G[0]->dmax_cnt;
        double mn = G[0]->dmin_traj[0], mx = G[0]->dmax_traj[0];
        for (int i = 1; i < count; ++i) {
            for (size_t c = 0; c < mins.size(); ++c) {
                mins[c] = std::min(mins[c], G[i]->dmin_cnt[c]);
                maxs[c] = std::max(maxs[c], G[i]->dmax_cnt[c]);
            }
            mn = std::min(mn, G[i]->dmin_traj[0]); mx = std::max(mx, G[i]->dmax_traj[0]);
        }
        for (Plan* P : G) { P->dmin_cnt = mins; P->dmax_cnt = maxs; P->dmin_traj[0] = mn; P->dmax_traj[0] = mx; }
    }
    for (Plan* P : G) { P->tay.w_knot.clear(); P->group = G; }
    PB200_CATCH
}

int pb200_shards_propagate(pb200_plan** plans, int32_t count, double t_start, double t_stop, const pb200_run_opts* o,
                           pb200_run_stats* stats) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_shards_propagate");
    const std::vector<Plan*> G = shard_group(plans, count, "pb200_shards_propagate");
    if (o && ((o->integrator != 0 && o->integrator != 3) || o->max_step_samples > 0 || o->tol < 0.0))
        fail(PB200_ERR_UNSUPPORTED, "pb200_shards_propagate: shards run the Taylor propagator only (integrator 0 or 3, "
                                    "max_step_samples = 0, tol >= 0)");
    for (int r = 0; r < count; ++r)
        if (!G[r]->state_set) fail(PB200_ERR_STATE, "pb200_shards_propagate: no state set on shard %d", r);
    Plan& P0 = *G[0];
    const double tlo = P0.times.front(), thi = P0.times.back(), eps = 1e-12;
    if (t_start < tlo - eps || t_stop > thi + eps || t_stop < t_start)
        fail(PB200_ERR_INVALID, "pb200_shards_propagate: [%g, %g] outside sampling times [%g, %g]", t_start, t_stop, tlo, thi);
    t_start = std::max(t_start, tlo); t_stop = std::min(t_stop, thi);
    PassGeom geo;
    bool tiled = false;
    taylor_geometry(P0, geo, tiled);
    // host half: the whole call, before any launch
    TaylorScheduler S(P0, t_start, t_stop, o);
    std::vector<TaylorStep> steps;
    for (TaylorStep s; S.next(s);) steps.push_back(s);
    int need = 0;
    for (const TaylorStep& s : steps) need = std::max(need, s.ring());
    // every shard's ring for the largest step, before the first launch: a ring that does not fit leaves the state as it was
    for (Plan* P : G) {
        CUDA_CHECK(cudaSetDevice(P->desc.device));
        try {
            taylor_grow_ring(*P, need);
        } catch (const Error& e) {
            fail(PB200_ERR_CUDA, "pb200_shards_propagate: this call needs the state and %d more state-sized buffers per shard, "
                                 "%lld bytes each (%d amplitudes x 16 B) besides the 8 B/amplitude interaction diagonal: %s",
                 need, (long long)(16 * P->D), (int)P->D, e.what());
        }
    }
    long long launches = 0;
    size_t i = 0;
    auto next = [&](TaylorStep& s) {
        if (i == steps.size()) return false;
        s = steps[i++];
        return true;
    };
    const float ms = taylor_launch_steps(G, geo, tiled, next, launches);
    if (stats) *stats = S.finish(ms, launches);
    PB200_CATCH
}

int pb200_shards_apply_h(pb200_plan** plans, int32_t count, double t_us, const double* in, double* out) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_shards_apply_h");
    if (!in || !out) fail(PB200_ERR_INVALID, "null argument");
    const std::vector<Plan*> G = shard_group(plans, count, "pb200_shards_apply_h");
    std::vector<c2*> bin(count), bout(count);
    for (int r = 0; r < count; ++r) {
        Plan& P = *G[r];
        bin[r] = P.buf[(P.cur + 1) % 3].get(); bout[r] = P.buf[(P.cur + 2) % 3].get();
        CUDA_CHECK(cudaSetDevice(P.desc.device));
        CUDA_CHECK(cudaMemcpyAsync(bin[r], in + (size_t)2 * P.D * r, sizeof(c2) * (size_t)P.D, cudaMemcpyHostToDevice, P.stream));
    }
    shards_apply_h(G, t_us, bin, bout);
    for (int r = 0; r < count; ++r) {
        Plan& P = *G[r];
        CUDA_CHECK(cudaSetDevice(P.desc.device));
        CUDA_CHECK(cudaMemcpyAsync(out + (size_t)2 * P.D * r, bout[r], sizeof(c2) * (size_t)P.D, cudaMemcpyDeviceToHost, P.stream));
    }
    shards_sync(G);
    PB200_CATCH
}

int pb200_shards_energy(pb200_plan** plans, int32_t count, double t_us, double* energy, double* h2) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_shards_energy");
    if (!energy || !h2) fail(PB200_ERR_INVALID, "null argument");
    const std::vector<Plan*> G = shard_group(plans, count, "pb200_shards_energy");
    std::vector<c2*> psi(count), hpsi(count);
    for (int r = 0; r < count; ++r) {
        if (!G[r]->state_set) fail(PB200_ERR_STATE, "pb200_shards_energy: no state set on shard %d", r);
        psi[r] = G[r]->buf[G[r]->cur].get(); hpsi[r] = G[r]->buf[(G[r]->cur + 2) % 3].get();
    }
    shards_apply_h(G, t_us, psi, hpsi);
    // Re<psi, H psi> and <H psi, H psi>, summed over the shards
    double e = 0.0, e2 = 0.0;
    for (int r = 0; r < count; ++r) {
        Plan& P = *G[r];
        CUDA_CHECK(cudaSetDevice(P.desc.device));
        const long long blocks = std::min<long long>((P.D + 255) / 256, (long long)P.sm_count * 8);
        double acc[2];
        device_sum(P, P.d_scratch.get(), 2, acc, [&] {
            dot2_kernel<<<dim3((unsigned)std::max<long long>(blocks, 1), 1), 256, 0, P.stream>>>(psi[r], hpsi[r], P.D,
                                                                                                 P.d_scratch.get());
        });
        e += acc[0]; e2 += acc[1];
    }
    energy[0] = e; h2[0] = e2;
    PB200_CATCH
}

int pb200_shards_expect(pb200_plan** plans, int32_t count, const pb200_op_terms* op, double* out) {
    PB200_TRY
    NvtxRange nvtx_range("pb200_shards_expect");
    if (!out) fail(PB200_ERR_INVALID, "pb200_shards_expect: null argument");
    const std::vector<Plan*> G = shard_group(plans, count, "pb200_shards_expect");
    const Plan& P0 = *G[0];
    check_op_terms(op, P0.n, P0.dim, "pb200_shards_expect");
    for (int r = 0; r < count; ++r)
        if (!G[r]->state_set) fail(PB200_ERR_STATE, "pb200_shards_expect: no state set on shard %d", r);
    out[0] = out[1] = 0.0;
    const int L = P0.n - P0.shard_bits;
    const ExpHost H = exp_host(op, P0.n, P0.dim, L);
    if (H.n_chunks == 0) return PB200_OK;
    // shard r reads shard r ^ x for every shard-bit pattern x the masks use: peer access where their devices differ
    // (pb200_shards_link enables only the single-bit pairs)
    for (int x = 1; x < count; ++x) {
        if (!((H.used_shard_bits >> x) & 1u)) continue;
        for (int r = 0; r < count; ++r) {
            const int di = G[r]->desc.device, dj = G[r ^ x]->desc.device;
            if (di == dj) continue;
            int can = 0;
            CUDA_CHECK(cudaDeviceCanAccessPeer(&can, di, dj));
            if (!can)
                fail(PB200_ERR_UNSUPPORTED, "pb200_shards_expect: the operator pairs shards %d and %d, but device %d cannot "
                                            "access the memory of device %d (no peer access)", r, r ^ x, di, dj);
            CUDA_CHECK(cudaSetDevice(di));
            const cudaError_t e = cudaDeviceEnablePeerAccess(dj, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
            else CUDA_CHECK(e);
        }
    }
    ExpSrc src{};
    src.local_bits = L;
    for (int r = 0; r < count; ++r) src.p[r] = G[r]->buf[G[r]->cur].get();
    std::vector<DevBuf<char>> X(count);
    std::vector<DevBuf<double>> acc(count);
    // every shard's kernel reads its peers' slices: all streams are idle before any buffer of the group is released
    struct GroupIdle {
        const std::vector<Plan*>& G;
        ~GroupIdle() {
            for (Plan* P : G)
                if (cudaStreamSynchronize(P->stream) != cudaSuccess) cudaGetLastError();
        }
    } idle{G};
    shards_sync(G);  // every slice is complete before a shard reads a peer's
    for (int r = 0; r < count; ++r) {
        Plan& P = *G[r];
        CUDA_CHECK(cudaSetDevice(P.desc.device));
        X[r] = upload_exp(H, P);
        acc[r].reset(P, 2);
        src.shard = r;
        sum_launch(P, acc[r].get(), 2, [&] { launch_expect<false>(P, P.D, H, X[r].get(), src, nullptr, 1, acc[r].get()); });
    }
    for (int r = 0; r < count; ++r) {
        double a[2];
        CUDA_CHECK(cudaSetDevice(G[r]->desc.device));
        sum_fetch(*G[r], acc[r].get(), 2, a);
        out[0] += a[0]; out[1] += a[1];
    }
    shards_sync(G);  // no shard still reads a peer's slice
    PB200_CATCH
}

int pb200_host_interpolate(const double* x, const double* y, int32_t n, int32_t order, const double* tq, int32_t nq,
                           double* out) {
    PB200_TRY
    if (!x || !y || !tq || !out || n < 2) fail(PB200_ERR_INVALID, "bad argument");
    std::vector<double> xs(x, x + n);
    auto pc = make_interpolant<cplx>(x, reinterpret_cast<const cplx*>(y), n, order);
    for (int i = 0; i < nq; ++i) {
        const cplx v = eval_at(pc, xs, tq[i], order);
        out[2 * i] = v.real(); out[2 * i + 1] = v.imag();
    }
    PB200_CATCH
}

int pb200_host_moments(const double* x, const double* y, int32_t n, int32_t order, double a, double b, double* out4) {
    PB200_TRY
    if (!x || !y || !out4 || n < 2) fail(PB200_ERR_INVALID, "bad argument");
    std::vector<double> xs(x, x + n);
    auto pc = make_interpolant<cplx>(x, reinterpret_cast<const cplx*>(y), n, order);
    cplx b0, b1;
    magnus_moments(pc, xs, a, b, b0, b1);
    out4[0] = b0.real(); out4[1] = b0.imag(); out4[2] = b1.real(); out4[3] = b1.imag();
    PB200_CATCH
}

int pb200_host_taylor_fit(const double* x, const double* y, int32_t n, int32_t order, double a, double h, int32_t p,
                          double* coeffs, double* resid) {
    PB200_TRY
    if (!x || !y || !coeffs || n < 2 || p < 0 || p > PB200_TAYLOR_PMAX || !(h > 0.0)) fail(PB200_ERR_INVALID, "bad argument");
    std::vector<double> xs(x, x + n);
    auto pc = make_interpolant<double>(x, y, n, order);
    const TaylorPoly f = taylor_fit(pc, xs, order, a, h, p);
    for (int i = 0; i <= p; ++i) coeffs[i] = f.c[i];
    if (resid) *resid = f.resid;
    PB200_CATCH
}

int pb200_host_taylor_separable(const double* coef, const double* det, int32_t n_traj, int32_t n_qudits, int32_t n_times,
                                int32_t* separable, double* a_out, double* c_out, double* m_out) {
    PB200_TRY
    if (!coef || !det || !separable || n_traj < 1 || n_qudits < 1 || n_times < 2) fail(PB200_ERR_INVALID, "bad argument");
    const cplx* y = reinterpret_cast<const cplx*>(coef);
    const size_t nt = (size_t)n_times, N = (size_t)n_qudits;
    const SeparableFit F = taylor_separable(
        n_traj, n_qudits, n_times, [&](int b, int k, int i) { return y[((size_t)b * N + k) * nt + i]; },
        [&](int b, int k, int i) { return det[((size_t)b * N + k) * nt + i]; });
    *separable = F.ok ? 1 : 0;
    if (F.ok) {
        // the factors refer to the reference row: report them scaled by its phase so that coef = a x |ref row| shape
        if (a_out)
            for (size_t x = 0; x < F.a.size(); ++x) { a_out[2 * x] = F.a[x].real(); a_out[2 * x + 1] = F.a[x].imag(); }
        if (c_out) for (size_t x = 0; x < (size_t)n_traj * N; ++x) c_out[x] = F.ns ? F.c[x] : 0.0;
        if (m_out) for (size_t i = 0; i < nt; ++i) m_out[i] = F.ns ? F.m[0][i] : 0.0;
    }
    PB200_CATCH
}

int pb200_host_taylor_shapes(const double* coef, const double* det, int32_t n_traj, int32_t n_qudits, int32_t n_times,
                             int32_t max_shapes, int32_t* n_shapes, double* a_out, double* c_out, double* m_out) {
    PB200_TRY
    if (!coef || !det || !n_shapes || n_traj < 1 || n_qudits < 1 || n_times < 2 || max_shapes < 0 ||
        max_shapes > PB200_TAYLOR_SMAX)
        fail(PB200_ERR_INVALID, "bad argument");
    const cplx* y = reinterpret_cast<const cplx*>(coef);
    const size_t nt = (size_t)n_times, N = (size_t)n_qudits, S = (size_t)max_shapes;
    const SeparableFit F = taylor_separable(
        n_traj, n_qudits, n_times, [&](int b, int k, int i) { return y[((size_t)b * N + k) * nt + i]; },
        [&](int b, int k, int i) { return det[((size_t)b * N + k) * nt + i]; }, max_shapes);
    *n_shapes = F.ok ? F.ns : -1;
    if (F.ok) {
        if (a_out)
            for (size_t x = 0; x < F.a.size(); ++x) { a_out[2 * x] = F.a[x].real(); a_out[2 * x + 1] = F.a[x].imag(); }
        if (c_out)
            for (size_t x = 0; x < (size_t)n_traj * N; ++x)
                for (size_t s = 0; s < S; ++s) c_out[x * S + s] = (int)s < F.ns ? F.c[x * F.ns + s] : 0.0;
        if (m_out)
            for (size_t s = 0; s < S; ++s)
                for (size_t i = 0; i < nt; ++i) m_out[s * nt + i] = (int)s < F.ns ? F.m[s][i] : 0.0;
    }
    PB200_CATCH
}

int pb200_host_taylor_order(double h, const double* m, int32_t p, double tol, int32_t* order_out, double* tail_out) {
    PB200_TRY
    if (!m || !order_out || p < 0 || p > PB200_TAYLOR_PMAX) fail(PB200_ERR_INVALID, "bad argument");
    double tail = 0.0;
    *order_out = taylor_order(h, std::vector<double>(m, m + p + 1), tol, tail);
    if (tail_out) *tail_out = tail;
    PB200_CATCH
}

int pb200_host_taylor_lowprec(double h, const double* m, int32_t p, int32_t K, int32_t g_stored, double tol,
                              int32_t* k_lo_out, double* bound_out) {
    PB200_TRY
    if (!m || !k_lo_out || p < 0 || p > PB200_TAYLOR_PMAX || K < 1) fail(PB200_ERR_INVALID, "bad argument");
    double bound = 0.0;
    *k_lo_out = taylor_lowprec_order(h, std::vector<double>(m, m + p + 1), K, g_stored != 0, tol, bound);
    if (bound_out) *bound_out = bound;
    PB200_CATCH
}

int pb200_host_chebyshev(double rho, double tol, double* out, int32_t cap, int32_t* count) {
    PB200_TRY
    if (!out || !count) fail(PB200_ERR_INVALID, "bad argument");
    std::vector<cplx> a = chebyshev_exp_coeffs(rho, tol);
    *count = (int32_t)a.size();
    for (int i = 0; i < (int)a.size() && i < cap; ++i) { out[2 * i] = a[i].real(); out[2 * i + 1] = a[i].imag(); }
    PB200_CATCH
}

}  // extern "C"
