// sm_90a (H100) kernels of the matrix-free propagator.
//
// Hot op (one Clenshaw stage of the Chebyshev expansion of exp(-iG)):
//     out[s] = c_psi*psi[s] + c_b2*b2[s] + c_g * (Gt v)[s]
//     (Gt v)[s] = (w*Dint[s] - sum_k th_k [digit_k(s)==from] - gamma) v[s]
//               + sum_k ( digit_k(s)==to ? g_k : conj(g_k) ) v[s with digit_k swapped]
// which restates, matrix-free, the CSR products QuTiP performs for the QobjEvo
// built at pulser-simulation/pulser_simulation/hamiltonian.py:246-439
// (SURVEY.md Appendix A.3).  HBM/L2-bound: algorithmic traffic is
// 16 (v) + 8 (Dint) + 16 (out) = 40 B per amplitude per apply.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

namespace pb200 {

struct c2 { double x, y; };

__host__ __device__ inline c2 cmul(c2 a, c2 b) { return {a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x}; }
__host__ __device__ inline c2 cadd(c2 a, c2 b) { return {a.x + b.x, a.y + b.y}; }

// ---- tile geometry of one pass -------------------------------------------
// A tile gathers the amplitudes whose index differs only in the bits
// [0, lo_bits) and [hi_shift, hi_shift + hi_bits); it is closed under flips of
// those bits, so their partners are served from shared memory.  Bits in
// `extra_mask` are flipped through coalesced global loads.
struct PassGeom {
    int n_bits;      // N (d = 2)
    int lo_bits;     // contiguous low bits in the tile (row = 2^lo_bits amps)
    int hi_shift;    // first bit of the high group
    int hi_bits;     // bits in the high group (rows = 2^hi_bits)
    uint32_t tile_flip_mask;   // tile-local bit positions whose flips belong to this pass
    unsigned long long extra_mask;  // global bit positions flipped via global loads
    int first_pass;  // 1: psi, b2 and the diagonal are added in this pass
};

struct StageCoef {  // complex scalars of the Clenshaw stage
    c2 c_psi, c_b2, c_g;
};

struct UniformDrive {  // same coefficients on every qubit and trajectory
    c2 g;          // scaled drive  g/rho
    double theta;  // scaled detuning moment
    double w;      // scaled weight of Dint
    double gamma;  // scaled centre
    int to_bit;    // digit value of |to> (1 for ground-rydberg / digital)
    int from_count_is_popc;  // 1: [digit==from] counted by popc(idx) (from digit = 1)
};

// per-(exponential, trajectory) table for non-uniform drives, d = 2:
//   tab[0 .. 2N)      g (re, im) per BIT position p
//   tab[2N .. 3N)     theta per bit position p
//   tab[3N], tab[3N+1] w, gamma
__host__ __device__ inline int d2_table_stride(int n) { return 3 * n + 2; }

// ---- PTX helpers: mbarrier + TMA 1-D bulk copy ----------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// TMA bulk copy global -> shared, completion signalled on the mbarrier
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

// streaming (read-once) 16-byte load / store
__device__ __forceinline__ c2 ld_stream(const c2* p) {
    double2 r = __ldcs(reinterpret_cast<const double2*>(p));
    return {r.x, r.y};
}
__device__ __forceinline__ void st_c2(c2* p, c2 v) {
    *reinterpret_cast<double2*>(p) = make_double2(v.x, v.y);
}
// 16-byte store whose L2 lines are evicted after the evict-normal / evict-first ones: for a result the next launch
// gathers from, while the launch streams more than the L2 holds
__device__ __forceinline__ void st_c2_evict_last(c2* p, c2 v) {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("st.global.L2::cache_hint.v2.f64 [%0], {%1, %2}, %3;" ::"l"(p), "d"(v.x), "d"(v.y), "l"(pol) : "memory");
}
// single-precision copies of an amplitude (the tail orders of a Taylor step): 8-byte stores, rounded to nearest
__device__ __forceinline__ void st_c2(float2* p, c2 v) { *p = make_float2((float)v.x, (float)v.y); }
__device__ __forceinline__ void st_c2_evict_last(float2* p, c2 v) {
    uint64_t pol;
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    asm volatile("st.global.L2::cache_hint.v2.f32 [%0], {%1, %2}, %3;" ::"l"(p), "f"((float)v.x), "f"((float)v.y), "l"(pol)
                 : "memory");
}
// an amplitude of a tile in shared memory or a gathered partner, in either precision, widened to fp64
__device__ __forceinline__ c2 tile_c2(const c2& t) { return t; }
__device__ __forceinline__ c2 tile_c2(const float2& t) { return {(double)t.x, (double)t.y}; }
__device__ __forceinline__ double2 ld_partner(const c2* p) { return __ldg(reinterpret_cast<const double2*>(p)); }
__device__ __forceinline__ double2 ld_partner(const float2* p) {
    const float2 r = __ldg(p);
    return make_double2((double)r.x, (double)r.y);
}

// Fused Lanczos step (StageArgs::lz set).  The gather source `v` holds the RAW vector r_j = G v_j - beta_{j-1} v_{j-1}
// of the previous stage; alpha_j = Re<v_j, r_j> and |r_j|^2 were reduced by that stage into lz.acc_prev.  This stage
//   v_{j+1} = (r_j - alpha_j v_j) / beta_j                           (second output, own element)
//   r_{j+1} = G v_{j+1} - beta_j v_j
//           = [G r_j - alpha_j r_j - alpha_j beta_{j-1} v_{j-1}] / beta_j - beta_j v_j     (G v_j = r_j + beta_{j-1} v_{j-1})
// so the separate vector-update kernel (48 B/amplitude, one launch per iteration) disappears: 88 B/amplitude per
// Lanczos iteration instead of 104, one launch.  Reference call replaced: qutip.sesolve, simulation.py:729-735.
struct LanczosFuse {
    const c2* vj;            // v_j      [B][D] own element
    const c2* vjm1;          // v_{j-1}  [B][D] own element (nullptr for j = 0)
    c2* vout;                // v_{j+1}  [B][D]
    const double* acc_prev;  // [B][2]: alpha_j, |r_j|^2
    const double* beta_prev; // [B]: beta_{j-1} (nullptr for j = 0)
    double* alpha_out;       // [B]: alpha_j recorded for the host
    double* beta_out;        // [B]: beta_j
    double* acc_clear;       // [B][2]: accumulator of the stage after this one, cleared here
};

struct LanczosCoef { double alpha, beta, inv, beta_prev; };

__device__ __forceinline__ LanczosCoef lanczos_coef(const LanczosFuse& lz, long long traj) {
    LanczosCoef c;
    c.alpha = lz.acc_prev[2 * traj];
    const double ww = lz.acc_prev[2 * traj + 1];
    const double b2 = ww - c.alpha * c.alpha;
    c.beta = (b2 > 1e-28 * fmax(ww, 1e-300)) ? sqrt(b2) : 0.0;   // 0: breakdown (invariant subspace reached)
    c.inv = c.beta > 0.0 ? 1.0 / c.beta : 0.0;
    c.beta_prev = lz.beta_prev ? lz.beta_prev[traj] : 0.0;
    return c;
}

// ---- d = 2 tiled stage kernel ---------------------------------------------
struct StageArgs {
    const c2* v;      // gather source      [B][D]
    const c2* psi;    // own element        [B][D]
    const c2* b2;     // own element        [B][D] (may alias out)
    c2* out;          // [B][D]
    const double* dint;        // [Bd][D]
    long long dint_stride;     // 0 when shared by all trajectories
    long long D;               // 2^N
    PassGeom geo;
    StageCoef coef;
    UniformDrive u;            // used when UNIFORM
    const double* table;       // [B][stride] for this exponential (non-uniform)
    int to_bit;
    int from_is_one;
    const double* beta_dev;  // Lanczos: c_b2 = -beta_dev[traj] read on the device (nullptr: use coef.c_b2)
    double* dot_acc;         // Lanczos: if set, acc[traj][0] += Re<lhs, out>, acc[traj][1] += <out, out> (fused reductions;
                             // lhs = v, or v_{j+1} in a fused Lanczos step)
    LanczosFuse lz;          // fused Lanczos step when lz.vj != nullptr (register-blocked kernels)
    // partner-sum forwarding (stage_d2_fwd_kernel, uniform drives): w_in[s] = sum of v over the flips this stage
    // does NOT perform (its producer's tile was closed under them), w_out[s] = the same sum of `out` over THIS
    // stage's tile flips for the consumer.  Plane 0 ([D]) holds P = sum v[s^k]; plane 1 (at + D * n_traj) holds the
    // signed sum Q a complex drive also needs.  Both may be null (first stage of a chain / nobody follows).
    const c2* w_in;
    c2* w_out;
    long long w_plane;       // distance between the P and the Q plane
};

// up to two independent Clenshaw chains per launch (the h and the h/2 branches of a Richardson step):
// blockIdx.y = chain * n_traj + trajectory
struct StageArgs2 {
    StageArgs a[2];
    int n_traj;
};

template <bool UNIFORM, bool REAL_G>
__global__ void __launch_bounds__(256) stage_d2_kernel(StageArgs a) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    c2* tile = reinterpret_cast<c2*>(smem_raw);
    __shared__ __align__(8) uint64_t mbar;

    const PassGeom g = a.geo;
    const int tbits = g.lo_bits + g.hi_bits;
    const int tsize = 1 << tbits;
    const long long traj = blockIdx.y;
    const long long tile_id = blockIdx.x;
    // bits of tile_id fill positions [lo, hi_shift) and [hi_shift + hi_bits, N)
    const int mid_bits = g.hi_shift - g.lo_bits;
    const long long mid = tile_id & ((1LL << mid_bits) - 1);
    const long long top = tile_id >> mid_bits;
    const long long base = (mid << g.lo_bits) | (top << (g.hi_shift + g.hi_bits));
    const long long voff = traj * a.D;
    const c2* vsrc = a.v + voff;

    // per-bit tables for non-uniform drives live after the tile
    double* tab = reinterpret_cast<double*>(tile + tsize);
    if (!UNIFORM) {
        const int stride = d2_table_stride(g.n_bits);
        const double* src = a.table + traj * stride;
        for (int i = threadIdx.x; i < stride; i += blockDim.x) tab[i] = src[i];
    }

    if (threadIdx.x == 0) mbar_init(&mbar, 1);
    __syncthreads();
    if (threadIdx.x == 0) mbar_arrive_expect_tx(&mbar, (uint32_t)tsize * 16u);
    {
        const int rows = 1 << g.hi_bits;
        const uint32_t row_bytes = (uint32_t)(16u << g.lo_bits);
        for (int r = threadIdx.x; r < rows; r += blockDim.x)
            tma_load_1d(tile + ((size_t)r << g.lo_bits), vsrc + base + ((long long)r << g.hi_shift), row_bytes, &mbar);
    }
    mbar_wait(&mbar, 0);

    const long long lomask = (1LL << g.lo_bits) - 1;
    double w, gamma, theta_u;
    c2 gu;
    if (UNIFORM) {
        w = a.u.w; gamma = a.u.gamma; theta_u = a.u.theta; gu = a.u.g;
    } else {
        w = tab[3 * g.n_bits]; gamma = tab[3 * g.n_bits + 1]; theta_u = 0.0; gu = {0.0, 0.0};
    }
    const int to_bit = a.to_bit;

    for (int t = threadIdx.x; t < tsize; t += blockDim.x) {
        const long long idx = base | (t & lomask) | ((long long)(t >> g.lo_bits) << g.hi_shift);
        const c2 vo = tile[t];
        double pr = 0.0, pi = 0.0, qr = 0.0, qi = 0.0;  // uniform: P, Q sums; non-uniform: pr,pi = drive result
        // flips served from shared memory
#pragma unroll 1
        for (uint32_t m = g.tile_flip_mask; m; m &= m - 1) {
            const int j = __ffs(m) - 1;
            const c2 pv = tile[t ^ (1 << j)];
            const int bit = (t >> j) & 1;
            if (UNIFORM) {
                pr += pv.x; pi += pv.y;
                if (!REAL_G) {
                    const double s = (bit == to_bit) ? 1.0 : -1.0;
                    qr = fma(s, pv.x, qr); qi = fma(s, pv.y, qi);
                }
            } else {
                const int p = (j < g.lo_bits) ? j : (j - g.lo_bits + g.hi_shift);
                const double gx = tab[2 * p];
                const double gy = (bit == to_bit) ? tab[2 * p + 1] : -tab[2 * p + 1];
                pr = fma(gx, pv.x, pr); pr = fma(-gy, pv.y, pr);
                pi = fma(gx, pv.y, pi); pi = fma(gy, pv.x, pi);
            }
        }
        // flips served by coalesced global loads
#pragma unroll 1
        for (unsigned long long m = g.extra_mask; m; m &= m - 1) {
            const int p = __ffsll((long long)m) - 1;
            const double2 raw = __ldg(reinterpret_cast<const double2*>(vsrc + (idx ^ (1LL << p))));
            const c2 pv = {raw.x, raw.y};
            const int bit = (int)((idx >> p) & 1);
            if (UNIFORM) {
                pr += pv.x; pi += pv.y;
                if (!REAL_G) {
                    const double s = (bit == to_bit) ? 1.0 : -1.0;
                    qr = fma(s, pv.x, qr); qi = fma(s, pv.y, qi);
                }
            } else {
                const double gx = tab[2 * p];
                const double gy = (bit == to_bit) ? tab[2 * p + 1] : -tab[2 * p + 1];
                pr = fma(gx, pv.x, pr); pr = fma(-gy, pv.y, pr);
                pi = fma(gx, pv.y, pi); pi = fma(gy, pv.x, pi);
            }
        }
        c2 drive;
        if (UNIFORM) {
            // g*S_to + conj(g)*S_from = x*P + i*y*Q
            drive.x = gu.x * pr; drive.y = gu.x * pi;
            if (!REAL_G) { drive.x = fma(-gu.y, qi, drive.x); drive.y = fma(gu.y, qr, drive.y); }
        } else {
            drive = {pr, pi};
        }
        c2 res;
        if (g.first_pass) {
            double diag = -gamma;
            if (a.dint) diag = fma(w, __ldcs(a.dint + traj * a.dint_stride + idx), diag);
            if (UNIFORM) {
                const int ones = __popcll((unsigned long long)idx);
                const int cnt = a.from_is_one ? ones : (g.n_bits - ones);
                diag = fma(-theta_u, (double)cnt, diag);
            } else {
                double acc = 0.0;
                for (int p = 0; p < g.n_bits; ++p) {
                    const int bit = (int)((idx >> p) & 1);
                    acc += (bit == a.from_is_one) ? tab[2 * g.n_bits + p] : 0.0;
                }
                diag -= acc;
            }
            c2 gv = {fma(diag, vo.x, drive.x), fma(diag, vo.y, drive.y)};
            res = cmul(a.coef.c_g, gv);
            if (a.psi) res = cadd(res, cmul(a.coef.c_psi, ld_stream(a.psi + voff + idx)));
            if (a.b2) res = cadd(res, cmul(a.beta_dev ? c2{-a.beta_dev[traj], 0.0} : a.coef.c_b2, ld_stream(a.b2 + voff + idx)));
        } else {
            res = cadd(ld_stream(a.out + voff + idx), cmul(a.coef.c_g, drive));
        }
        st_c2(a.out + voff + idx, res);
    }
}

// ---- d = 2 tiled stage kernel, register-blocked (the production kernel) ------
// Each thread owns R = 2^RB amplitudes of the tile (tile index t = tid + r*NT,
// i.e. the top RB tile bits live in registers): flips of those bits are
// register-to-register, flips of the other tile bits cost one LDS.128 per owned
// amplitude, all independent (fully unrolled) so that the shared-memory pipe
// stays full.  Shared-memory operand traffic per amplitude and pass is
// (flipped tile bits - RB + 1) x 16 B.
// Compute phase of one tile, shared by the one-shot and the persistent kernels: gathers from the tile in
// shared memory (register-blocked), optional global-load partners, fused epilogue and store.
// own-element global load: streaming (read once per stage)
__device__ __forceinline__ c2 ld_own(const c2* p) {
    double2 r = __ldcs(reinterpret_cast<const double2*>(p));
    return {r.x, r.y};
}
__device__ __forceinline__ c2 ld_own(const float2* p) {
    const float2 r = __ldcs(p);
    return {(double)r.x, (double)r.y};
}

// one partner of a complex-drive Taylor stage: z = f chi (f = gx + i gy, the factor of the partner's transition),
// p += z, q += sg z
__device__ __forceinline__ void taylor_signed_add(double gx, double gy, double sg, double x, double y, double& pr, double& pi,
                                                  double& qr, double& qi) {
    const double zx = fma(gx, x, -gy * y), zy = fma(gx, y, gy * x);
    pr += zx; pi += zy;
    qr = fma(sg, zx, qr); qi = fma(sg, zy, qi);
}

// In-tile partner sums of the R = 2^RB amplitudes a thread owns (tile index t = tid + r*NT): flips of the
// register-block bits (tile bits TBITS-RB .. TBITS-1) are register moves, flips of the tile bits
// [jstart, TBITS-RB) are independent LDS.128 from `tile`.
// SIGNED (per-bit table only): q also receives the signed sum  sum_k sg_k f_k chi_k,  sg_k = +1 where the amplitude's bit
// k is to_bit, with f_k the factor p receives (the complex-drive Taylor stage).  COLSIGN: vec(rho) with a complex drive,
// sg_k is negated on the column bits (bit positions below ncol), whose y-factor is i conj(unit) rather than i unit.
// T: c2, or float2 for a single-precision tile (LDS.64).
template <bool UNIFORM, bool REAL_G, int TBITS, int RB, bool SIGNED = false, bool COLSIGN = false, class T = c2>
__device__ __forceinline__ void rb_tile_gather(const PassGeom& g, const T* tile, const double* __restrict__ tab, int tid,
                                               int to_bit, int jstart, bool skip_smem, const c2 (&v)[1 << RB],
                                               double (&pr)[1 << RB], double (&pi)[1 << RB], double (&qr)[1 << RB],
                                               double (&qi)[1 << RB], int ncol = 0) {
    static_assert(!SIGNED || !UNIFORM, "signed sums of the per-bit table gather");
    static_assert(!COLSIGN || SIGNED, "the column sign belongs to the signed sums");
    constexpr int R = 1 << RB;
    constexpr int NT = 1 << (TBITS - RB);
    // --- flips inside the register block (tile bits TBITS-RB .. TBITS-1) ---
#pragma unroll
    for (int q = 0; q < RB; ++q) {
        const int j = TBITS - RB + q;
        double gx = 0.0, gyt = 0.0;
        bool col = false;
        if (!UNIFORM) {
            const int p = (j < g.lo_bits) ? j : (j - g.lo_bits + g.hi_shift);
            gx = tab[2 * p]; gyt = tab[2 * p + 1];
            col = COLSIGN && p < ncol;
        }
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const c2 pv = v[r ^ (1 << q)];
            const int bit = (r >> q) & 1;
            if (UNIFORM) {
                pr[r] += pv.x; pi[r] += pv.y;
                if (!REAL_G) {
                    if (bit == to_bit) { qr[r] += pv.x; qi[r] += pv.y; } else { qr[r] -= pv.x; qi[r] -= pv.y; }
                }
            } else if constexpr (SIGNED) {
                const double gy = (bit == to_bit) ? gyt : -gyt;
                taylor_signed_add(gx, gy, ((bit == to_bit) != col) ? 1.0 : -1.0, pv.x, pv.y, pr[r], pi[r], qr[r], qi[r]);
            } else {
                const double gy = (bit == to_bit) ? gyt : -gyt;
                pr[r] = fma(gx, pv.x, pr[r]); pr[r] = fma(-gy, pv.y, pr[r]);
                pi[r] = fma(gx, pv.y, pi[r]); pi[r] = fma(gy, pv.x, pi[r]);
            }
        }
    }
    // --- flips served from shared memory ---
#pragma unroll
    for (int j = 0; j < TBITS - RB; ++j) {
        if (j >= jstart && !skip_smem) {
            const int bit = (tid >> j) & 1;
            const int ptid = tid ^ (1 << j);
            double gx = 0.0, gy = 0.0;
            bool col = false;
            if (!UNIFORM) {
                const int p = (j < g.lo_bits) ? j : (j - g.lo_bits + g.hi_shift);
                gx = tab[2 * p];
                gy = (bit == to_bit) ? tab[2 * p + 1] : -tab[2 * p + 1];
                col = COLSIGN && p < ncol;
            }
            const double sg = ((bit == to_bit) != col) ? 1.0 : -1.0;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const c2 pv = tile_c2(tile[ptid + r * NT]);
                if (UNIFORM) {
                    pr[r] += pv.x; pi[r] += pv.y;
                    if (!REAL_G) { qr[r] = fma(sg, pv.x, qr[r]); qi[r] = fma(sg, pv.y, qi[r]); }
                } else if constexpr (SIGNED) {
                    taylor_signed_add(gx, gy, sg, pv.x, pv.y, pr[r], pi[r], qr[r], qi[r]);
                } else {
                    pr[r] = fma(gx, pv.x, pr[r]); pr[r] = fma(-gy, pv.y, pr[r]);
                    pi[r] = fma(gx, pv.y, pi[r]); pi[r] = fma(gy, pv.x, pi[r]);
                }
            }
        }
    }
}

// Compute phase of one tile: gathers from the tile in shared memory (register-blocked), coalesced global loads
// for the partners outside the tile, fused epilogue (diagonal, Clenshaw / Lanczos combination, reductions) and store.
template <bool UNIFORM, bool REAL_G, int TBITS, int RB>
__device__ __forceinline__ void rb_tile_compute(const StageArgs& a, const PassGeom& g, const c2* tile,
                                                const double* __restrict__ tab, long long base, long long traj,
                                                int tid, uint64_t* tile_bar) {
    constexpr int R = 1 << RB;
    constexpr int NT = 1 << (TBITS - RB);
    const long long voff = traj * a.D;
    const c2* vsrc = a.v + voff;
    const long long lomask = (1LL << g.lo_bits) - 1;
    const int to_bit = a.to_bit;
    // first tile bit whose flip belongs to this pass (pass A: 0, later passes: lo_bits)
    const int jstart = __ffs(g.tile_flip_mask) - 1;

    c2 v[R];
    double pr[R], pi[R], qr[R], qi[R];
    // global index of each owned amplitude
    long long idx[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        const int t = tid + r * NT;
        idx[r] = base | (t & lomask) | ((long long)(t >> g.lo_bits) << g.hi_shift);
        pr[r] = 0.0; pi[r] = 0.0; qr[r] = 0.0; qi[r] = 0.0;
    }
    // --- flips of the bits outside the tile: coalesced partner loads.  They do not depend on the tile, so they go
    //     out while the bulk copy of the tile is still in flight (the wait on its mbarrier comes after them) ---
    for (unsigned long long m = g.extra_mask; m; m &= m - 1) {
        const int p = __ffsll((long long)m) - 1;
        double gx = 0.0, gyt = 0.0;
        if (!UNIFORM) { gx = tab[2 * p]; gyt = tab[2 * p + 1]; }
        const int bit = (int)((base >> p) & 1);  // extra bits are never tile bits
        const double sg = (bit == to_bit) ? 1.0 : -1.0;
        const double gy = (bit == to_bit) ? gyt : -gyt;
        double2 raw[R];
#pragma unroll
        for (int r = 0; r < R; ++r) raw[r] = __ldg(reinterpret_cast<const double2*>(vsrc + (idx[r] ^ (1LL << p))));
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if (UNIFORM) {
                pr[r] += raw[r].x; pi[r] += raw[r].y;
                if (!REAL_G) { qr[r] = fma(sg, raw[r].x, qr[r]); qi[r] = fma(sg, raw[r].y, qi[r]); }
            } else {
                pr[r] = fma(gx, raw[r].x, pr[r]); pr[r] = fma(-gy, raw[r].y, pr[r]);
                pi[r] = fma(gx, raw[r].y, pi[r]); pi[r] = fma(gy, raw[r].x, pi[r]);
            }
        }
    }
    if (tile_bar) mbar_wait(tile_bar, 0);
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = tile[tid + r * NT];
    rb_tile_gather<UNIFORM, REAL_G, TBITS, RB>(g, tile, tab, tid, to_bit, jstart, false, v, pr, pi, qr, qi);
    // --- epilogue ---
    double w = 0.0, gamma = 0.0, th_common = 0.0;
    double th_r[R];
    if (g.first_pass) {
        if (UNIFORM) { w = a.u.w; gamma = a.u.gamma; }
        else {
            w = tab[3 * g.n_bits]; gamma = tab[3 * g.n_bits + 1];
            // theta sum split into (bits of base) + (bits of tid) + (register bits)
            const long long fixed = base | (tid & lomask) | ((long long)(tid >> g.lo_bits) << g.hi_shift);
            for (int p = 0; p < g.n_bits; ++p) {
                const int bit = (int)((fixed >> p) & 1);
                th_common += (bit == a.from_is_one) ? tab[2 * g.n_bits + p] : 0.0;
            }
#pragma unroll
            for (int r = 0; r < R; ++r) {
                double acc = 0.0;
#pragma unroll
                for (int q = 0; q < RB; ++q) {
                    const int j = TBITS - RB + q;
                    const int p = (j < g.lo_bits) ? j : (j - g.lo_bits + g.hi_shift);
                    // `fixed` has these bits at 0: replace the bit-0 contribution by the bit-(r>>q) one
                    const double th = tab[2 * g.n_bits + p];
                    const int bit = (r >> q) & 1;
                    acc += ((bit == a.from_is_one) ? th : 0.0) - ((0 == a.from_is_one) ? th : 0.0);
                }
                th_r[r] = acc;
            }
        }
    }
    // drive term of every owned amplitude (frees the P/Q accumulators)
#pragma unroll
    for (int r = 0; r < R; ++r) {
        if (UNIFORM) {
            const double dx = a.u.g.x * pr[r], dy = a.u.g.x * pi[r];
            if (!REAL_G) { pr[r] = fma(-a.u.g.y, qi[r], dx); pi[r] = fma(a.u.g.y, qr[r], dy); }
            else { pr[r] = dx; pi[r] = dy; }
        }
    }
    // own-element global operands are staged in registers half a block at a time so that the loads
    // of one half are all in flight together (the stores to `out` may alias them for the compiler)
    constexpr int H = (R >= 4) ? R / 2 : R;
    const c2 cb2 = a.beta_dev ? c2{-a.beta_dev[traj], 0.0} : a.coef.c_b2;
    const bool fuse = a.lz.vj != nullptr;
    LanczosCoef lc{0.0, 0.0, 0.0, 0.0};
    if (fuse) lc = lanczos_coef(a.lz, traj);
    double dot0 = 0.0, dot1 = 0.0;
    if (g.first_pass) {
        const double* dsrc = a.dint ? a.dint + traj * a.dint_stride : nullptr;
#pragma unroll
        for (int h0 = 0; h0 < R; h0 += H) {
            double dv[H];
            c2 pv[H], bv[H];
#pragma unroll
            for (int r = 0; r < H; ++r) {
                dv[r] = dsrc ? __ldcs(dsrc + idx[h0 + r]) : 0.0;
                if (fuse) {
                    pv[r] = ld_own(a.lz.vj + voff + idx[h0 + r]);
                    bv[r] = (a.lz.vjm1 && lc.beta_prev != 0.0) ? ld_own(a.lz.vjm1 + voff + idx[h0 + r]) : c2{0.0, 0.0};
                } else {
                    pv[r] = a.psi ? ld_own(a.psi + voff + idx[h0 + r]) : c2{0.0, 0.0};
                    bv[r] = a.b2 ? ld_own(a.b2 + voff + idx[h0 + r]) : c2{0.0, 0.0};
                }
            }
#pragma unroll
            for (int r = 0; r < H; ++r) {
                const int rr = h0 + r;
                double diag = fma(w, dv[r], -gamma);
                if (UNIFORM) {
                    const int ones = __popcll((unsigned long long)idx[rr]);
                    const int cnt = a.from_is_one ? ones : (g.n_bits - ones);
                    diag = fma(-a.u.theta, (double)cnt, diag);
                } else {
                    diag -= th_common + th_r[rr];
                }
                const c2 gv = {fma(diag, v[rr].x, pr[rr]), fma(diag, v[rr].y, pi[rr])};
                c2 res, lhs;
                if (fuse) {
                    // v_{j+1} and r_{j+1} from the raw vector (see LanczosFuse)
                    const c2 vn = {(v[rr].x - lc.alpha * pv[r].x) * lc.inv, (v[rr].y - lc.alpha * pv[r].y) * lc.inv};
                    const double ai = lc.alpha * lc.inv, abi = ai * lc.beta_prev;
                    res.x = fma(lc.inv, gv.x, -fma(ai, v[rr].x, fma(abi, bv[r].x, lc.beta * pv[r].x)));
                    res.y = fma(lc.inv, gv.y, -fma(ai, v[rr].y, fma(abi, bv[r].y, lc.beta * pv[r].y)));
                    st_c2(a.lz.vout + voff + idx[rr], vn);
                    lhs = vn;
                } else {
                    res = cmul(a.coef.c_g, gv);
                    res = cadd(res, cmul(a.coef.c_psi, pv[r]));
                    res = cadd(res, cmul(cb2, bv[r]));
                    lhs = v[rr];
                }
                dot0 = fma(lhs.x, res.x, dot0); dot0 = fma(lhs.y, res.y, dot0);
                dot1 = fma(res.x, res.x, dot1); dot1 = fma(res.y, res.y, dot1);
                st_c2(a.out + voff + idx[rr], res);
            }
        }
    } else {
#pragma unroll
        for (int h0 = 0; h0 < R; h0 += H) {
            c2 ov[H];
#pragma unroll
            for (int r = 0; r < H; ++r) ov[r] = ld_own(a.out + voff + idx[h0 + r]);
#pragma unroll
            for (int r = 0; r < H; ++r) {
                const int rr = h0 + r;
                const c2 res = cadd(ov[r], cmul(a.coef.c_g, c2{pr[rr], pi[rr]}));
                dot0 = fma(v[rr].x, res.x, dot0); dot0 = fma(v[rr].y, res.y, dot0);
                dot1 = fma(res.x, res.x, dot1); dot1 = fma(res.y, res.y, dot1);
                st_c2(a.out + voff + idx[rr], res);
            }
        }
    }
    if (a.dot_acc) {  // block reduction of the fused Lanczos inner products, one atomic pair per CTA
        for (int o = 16; o > 0; o >>= 1) {
            dot0 += __shfl_xor_sync(0xffffffffu, dot0, o);
            dot1 += __shfl_xor_sync(0xffffffffu, dot1, o);
        }
        __shared__ double dred[2][NT / 32 > 0 ? NT / 32 : 1];
        if ((tid & 31) == 0) { dred[0][tid >> 5] = dot0; dred[1][tid >> 5] = dot1; }
        __syncthreads();
        if (tid == 0) {
            double s0 = 0.0, s1 = 0.0;
#pragma unroll
            for (int i = 0; i < NT / 32; ++i) { s0 += dred[0][i]; s1 += dred[1][i]; }
            atomicAdd(a.dot_acc + 2 * traj, s0);
            atomicAdd(a.dot_acc + 2 * traj + 1, s1);
        }
    }
    if (fuse && blockIdx.x == 0 && tid == 0) {  // one CTA per trajectory records the recurrence coefficients
        a.lz.alpha_out[traj] = lc.alpha;
        a.lz.beta_out[traj] = lc.beta;
        a.lz.acc_clear[2 * traj] = 0.0;
        a.lz.acc_clear[2 * traj + 1] = 0.0;
    }
}

__device__ __forceinline__ long long tile_base_of(const PassGeom& g, long long tile_id) {
    // bits of tile_id fill positions [lo, hi_shift) and [hi_shift + hi_bits, N)
    const int mid_bits = g.hi_shift - g.lo_bits;
    const long long mid = tile_id & ((1LL << mid_bits) - 1);
    const long long top = tile_id >> mid_bits;
    return (mid << g.lo_bits) | (top << (g.hi_shift + g.hi_bits));
}

// programmatic dependent launch: wait for the producer grid's memory before the first global read
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- d = 2 tiled stage kernel, one tile per CTA --------------------------------
// Each thread owns R = 2^RB amplitudes of the tile (tile index t = tid + r*NT,
// i.e. the top RB tile bits live in registers): flips of those bits are
// register-to-register, flips of the other tile bits cost one LDS.128 per owned
// amplitude, all independent (fully unrolled) so that the shared-memory pipe
// stays full.  Shared-memory operand traffic per amplitude and pass is
// (flipped tile bits - RB + 1) x 16 B.
template <bool UNIFORM, bool REAL_G, int TBITS, int RB>
__global__ void __launch_bounds__(1 << (TBITS - RB), (65536 / ((1 << (TBITS - RB)) * (RB >= 3 ? 128 : 64))))
stage_d2_rb_kernel(const __grid_constant__ StageArgs2 m) {
    constexpr int NT = 1 << (TBITS - RB);
    constexpr int TSIZE = 1 << TBITS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    c2* tile = reinterpret_cast<c2*>(smem_raw);
    __shared__ __align__(8) uint64_t mbar;

    const int chain = blockIdx.y / m.n_traj;
    const StageArgs& a = m.a[chain];
    const PassGeom g = a.geo;
    const int tid = threadIdx.x;
    const long long traj = blockIdx.y - chain * m.n_traj;
    const long long base = tile_base_of(g, blockIdx.x);
    const c2* vsrc = a.v + traj * a.D;

    if (tid == 0) mbar_init(&mbar, 1);
    __syncthreads();          // the barrier is initialised before any thread issues a copy on it
    pdl_wait();
    pdl_launch_dependents();
    // the tile copy goes out first; the per-trajectory coefficient table (non-uniform drives) is read behind it
    if (tid == 0) mbar_arrive_expect_tx(&mbar, (uint32_t)TSIZE * 16u);
    const int rows = 1 << g.hi_bits;
    const uint32_t row_bytes = (uint32_t)(16u << g.lo_bits);
    for (int r = tid; r < rows; r += NT)
        tma_load_1d(tile + ((size_t)r << g.lo_bits), vsrc + base + ((long long)r << g.hi_shift), row_bytes, &mbar);
    double* tab = reinterpret_cast<double*>(tile + TSIZE);
    if (!UNIFORM) {
        const int stride = d2_table_stride(g.n_bits);
        const double* src = a.table + traj * stride;
        for (int i = tid; i < stride; i += NT) tab[i] = src[i];
        __syncthreads();
    }
    rb_tile_compute<UNIFORM, REAL_G, TBITS, RB>(a, g, tile, tab, base, traj, tid, &mbar);
}

// ---- d = 2 stage kernel with partner-sum forwarding (uniform drives) ---------------------------------------------
// The single-pass kernel above is bound by L2 throughput: (N - TBITS) x 16 B of partner loads per amplitude dominate
// its L2 sectors.  Here consecutive Clenshaw
// stages alternate between two tile geometries with complementary flip sets -- A: the TBITS low bits; B: the
// hb = min(N - TBITS, TBITS - 2) bits above them, gathered as 2^hb rows of 2^(TBITS - hb) amplitudes -- and a stage
// receives the partner sums over the OTHER geometry's flips from the stage that produced its input (w_in, 16 B per
// amplitude) and emits the sums of its own result over ITS flips (w_out): 104 B of L2 traffic per amplitude and stage
// instead of 72 + 16 (N - TBITS).  Bits above TBITS + hb (N > 20) stay coalesced partner loads in both geometries.
// Issuing the operand loads after the gathers leaves the kernel latency-bound, so every global operand of the stage
// is requested BEFORE the wait on the tile copy and folded into the
// accumulators as it arrives, so a CTA has one exposed memory latency.
template <bool REAL_G, int TBITS, int RB>
__global__ void __launch_bounds__(1 << (TBITS - RB), 2) stage_d2_fwd_kernel(const __grid_constant__ StageArgs2 m) {
    constexpr int R = 1 << RB;
    constexpr int NT = 1 << (TBITS - RB);
    constexpr int TSIZE = 1 << TBITS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    c2* tile = reinterpret_cast<c2*>(smem_raw);
    c2* rtile = tile + TSIZE;
    __shared__ __align__(8) uint64_t mbar;

    const int chain = blockIdx.y / m.n_traj;
    const StageArgs& a = m.a[chain];
    const PassGeom g = a.geo;
    const int tid = threadIdx.x;
    const long long traj = blockIdx.y - chain * m.n_traj;
    const long long base = tile_base_of(g, blockIdx.x);
    const long long voff = traj * a.D;
    const c2* vsrc = a.v + voff;

    if (tid == 0) mbar_init(&mbar, 1);
    __syncthreads();
    pdl_wait();
    pdl_launch_dependents();
    if (tid == 0) mbar_arrive_expect_tx(&mbar, (uint32_t)TSIZE * 16u);
    {
        const int rows = 1 << g.hi_bits;
        const uint32_t row_bytes = (uint32_t)(16u << g.lo_bits);
        for (int r = tid; r < rows; r += NT)
            tma_load_1d(tile + ((size_t)r << g.lo_bits), vsrc + base + ((long long)r << g.hi_shift), row_bytes, &mbar);
    }
    const long long lomask = (1LL << g.lo_bits) - 1;
    const long long fixed = base | (tid & lomask) | ((long long)(tid >> g.lo_bits) << g.hi_shift);
    // the register-block bits are the top RB tile bits: their global positions
    int pq[RB];
#pragma unroll
    for (int q = 0; q < RB; ++q) {
        const int j = TBITS - RB + q;
        pq[q] = (j < g.lo_bits) ? j : (j - g.lo_bits + g.hi_shift);
    }
    auto idx_of = [&](int r) {
        long long o = fixed;
#pragma unroll
        for (int q = 0; q < RB; ++q) o |= (long long)((r >> q) & 1) << pq[q];
        return o;
    };
    // ---- every global operand goes out now; each is folded into an accumulator as soon as it is used ----
    double pr[R], pi[R], qr[R], qi[R];
    c2 part[R];      // c_psi psi + c_b2 b2
    double dg[R];    // scaled diagonal of the amplitude
    {
        const double* dsrc = a.dint ? a.dint + traj * a.dint_stride : nullptr;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const long long ix = idx_of(r);
            c2 w0 = {0.0, 0.0}, w1 = {0.0, 0.0}, ps = {0.0, 0.0}, bb = {0.0, 0.0};
            if (a.w_in) { w0 = ld_own(a.w_in + voff + ix); if (!REAL_G) w1 = ld_own(a.w_in + a.w_plane + voff + ix); }
            if (a.psi) ps = ld_own(a.psi + voff + ix);
            if (a.b2) bb = ld_own(a.b2 + voff + ix);
            const double dv = dsrc ? __ldcs(dsrc + ix) : 0.0;
            pr[r] = w0.x; pi[r] = w0.y; qr[r] = w1.x; qi[r] = w1.y;
            part[r] = cadd(cmul(a.coef.c_psi, ps), cmul(a.coef.c_b2, bb));
            const int ones = __popcll((unsigned long long)ix);
            const int cnt = a.from_is_one ? ones : (g.n_bits - ones);
            dg[r] = fma(-a.u.theta, (double)cnt, fma(a.u.w, dv, -a.u.gamma));
        }
    }
    const int to_bit = a.to_bit;
    // partners across the bits above both geometries (N > TBITS + hb): coalesced loads, also ahead of the wait
    for (unsigned long long em = g.extra_mask; em; em &= em - 1) {
        const int p = __ffsll((long long)em) - 1;
        const double sg = (((base >> p) & 1) == to_bit) ? 1.0 : -1.0;
        double2 raw[R];
#pragma unroll
        for (int r = 0; r < R; ++r) raw[r] = __ldg(reinterpret_cast<const double2*>(vsrc + (idx_of(r) ^ (1LL << p))));
#pragma unroll
        for (int r = 0; r < R; ++r) {
            pr[r] += raw[r].x; pi[r] += raw[r].y;
            if (!REAL_G) { qr[r] = fma(sg, raw[r].x, qr[r]); qi[r] = fma(sg, raw[r].y, qi[r]); }
        }
    }
    mbar_wait(&mbar, 0);
    const int jstart = __ffs(g.tile_flip_mask) - 1;
    c2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = tile[tid + r * NT];
    rb_tile_gather<true, REAL_G, TBITS, RB>(g, tile, nullptr, tid, to_bit, jstart, false, v, pr, pi, qr, qi);
    // ---- epilogue: out = part + c_g (diag v + g (P + w_in)) ----
#pragma unroll
    for (int r = 0; r < R; ++r) {
        double dx = a.u.g.x * pr[r], dy = a.u.g.x * pi[r];
        if (!REAL_G) { dx = fma(-a.u.g.y, qi[r], dx); dy = fma(a.u.g.y, qr[r], dy); }
        const c2 gv = {fma(dg[r], v[r].x, dx), fma(dg[r], v[r].y, dy)};
        const c2 res = cadd(part[r], cmul(a.coef.c_g, gv));
        st_c2(a.out + voff + idx_of(r), res);
        v[r] = res;
    }
    if (a.w_out) {
        // sums of the RESULT over this tile's flips for the next stage (whose tile is not closed under them)
#pragma unroll
        for (int r = 0; r < R; ++r) {
            rtile[tid + r * NT] = v[r];
            pr[r] = 0.0; pi[r] = 0.0; qr[r] = 0.0; qi[r] = 0.0;
        }
        __syncthreads();
        rb_tile_gather<true, REAL_G, TBITS, RB>(g, rtile, nullptr, tid, to_bit, jstart, false, v, pr, pi, qr, qi);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const long long ix = idx_of(r);
            st_c2(a.w_out + voff + ix, c2{pr[r], pi[r]});
            if (!REAL_G) st_c2(a.w_out + a.w_plane + voff + ix, c2{qr[r], qi[r]});
        }
    }
}

// ---- d = 2 stage kernel of the time-dependent Taylor propagator (one drive time shape, its phase constant or moving) -
// On a step [a, a+h] the interpolated coefficients (QobjEvo's cubic splines, hamiltonian.py:436) are polynomials in
// u = (t-a)/h:  H(u) = sum_j H_j u^j,  H_0 = Dint - th_0 n_from - gam_0 + om_0 X,  H_j = -th_j n_from - gam_j + om_j X
// with X = sum_k (unit |to><from|_k + h.c.).  psi(u) = sum_k chi_k u^k solves psi' = -i h H(u) psi exactly when
//     (k+1) chi_{k+1} = -i h sum_{j <= min(p,k)} H_j chi_{k-j} ,
// i.e. ONE gather G_k = X chi_k per order and own-element history terms: no Magnus commutator error, no inner
// products, no host synchronisation; the step length is bounded by the spectral width (rho = h W, fp64
// cancellation: rho <= 14) and by the polynomial fit of the splines only.  The stage computes chi_{k+1} from the tile of chi_k,
// optionally stores G_k for later orders and folds chi_k + chi_{k+1} into the accumulator of psi(1) on every other
// order.  Replaces qutip.sesolve (simulation.py:729-735) for global drives (a phase that moves inside a step: the CPLX
// instantiations, two gathers per order), and -- with per-qubit
// static factors from a per-trajectory table (TaylorArgs::table) -- the trajectory loop's solves (simulation.py:885-915).
#define PB200_TAYLOR_PMAX 8
#define PB200_MAX_SHARD_BITS 3
#define PB200_TAYLOR_SMAX 4   // detuning time shapes with static per-qubit weights (detuning maps, masks, noise)
// table of a plan whose detuning has several shapes, or one shape on a uniform drive, per trajectory:
//   tab[0 .. 2N)              a unit (re, im) per BIT position p (the unit itself for a uniform drive)
//   tab[2N + s N + p]         weight c_s of bit position p, s < S
__host__ __device__ inline int taylor_table_stride(int n, int s) { return 2 * n + s * n; }
struct TaylorArgs {
    const c2* v;       // chi_k, gather source [B][D]
    c2* out;           // chi_{k+1}
    c2* g_out;         // G_k = X chi_k (nullptr: nobody reads it later)
    c2* acc;           // accumulator of sum_k chi_k
    const double* dint;  // Dint of the small kernel (nullptr: no interaction)
    long long dint_stride;  // 0: Dint shared by the trajectories
    // couplings of the tiled stage, which forms Dint itself (taylor_dint_setup): the symmetric N x N matrix U of
    // dint_kernel (atom i at bit position N - 1 - i, zero diagonal, bad atoms zeroed); nullptr: no interaction.  A pair
    // counts where both bits equal ryd_bit (the Rydberg digit)
    const double* cpl;
    long long cpl_stride;   // 0: shared by the trajectories, else N * N
    int ryd_bit;
    long long D;
    PassGeom geo;
    c2 unit;           // uniform drive: e^{-i phi}, the drive's phase on the step (TaylorStep::unit)
    // separable per-qubit drives (trajectory batches with static noise): coef_{b,k}(t) = a_{b,k} unit omega(t),
    // det_{b,k}(t) = theta(t) + c_{b,k} M(t).  table[b][0 .. 2N) = a unit per BIT position (re, im),
    // table[b][2N .. 3N) = c per bit position (layout of d2_table_stride); nullptr in the uniform case.
    // Several shapes, det_{b,k}(t) = theta(t) + sum_s c_{b,k,s} M_s(t): layout of taylor_table_stride(N, tab_shapes)
    const double* table;
    int tab_shapes;    // 0: d2_table_stride layout (one shape), else PB200_TAYLOR_SMAX (unused shapes have c = m = 0)
    int to_bit, from_is_one;
    double th0, gam0, om0;  // H_0 = Dint - th0 n_from - sum_s m0[s] sum_k c_{k,s} n_k - gam0 + om0 X
    double m0[PB200_TAYLOR_SMAX];
    c2 scale;          // -i h / (k+1)
    int nh;            // history terms j = 1 .. nh
    const c2* hchi[PB200_TAYLOR_PMAX];   // chi_{k-j}   (nullptr when th_j = m_j = gam_j = 0)
    const c2* hg[PB200_TAYLOR_PMAX];     // G_{k-j}     (nullptr when om_j = 0)
    double hth[PB200_TAYLOR_PMAX], hgam[PB200_TAYLOR_PMAX], hom[PB200_TAYLOR_PMAX];
    double hm[PB200_TAYLOR_SMAX][PB200_TAYLOR_PMAX];   // hm[s][j]: shape s, history j
    int acc_read;      // 1: acc is read before it is updated (0: first write of the step)
    int acc_add_v;     // 1: chi_k joins the update, 0: chi_{k+1} alone
    int acc_add_h;     // 1: chi_{k-1} (history term hchi[0]) joins the update as well
    int acc_on;        // 0: this order leaves the accumulator alone
    c2 acc_mul;        // factor of the whole accumulator (phase of the scalar centre on the last order, else 1)
    // precision of the order (TaylorStep::k_lo): chi_k (v) is single precision (float2 in the slot), chi_{k+1} and G_k
    // are stored so; bit j - 1 of hchi32 / hg32: chi_{k-j} / G_{k-j} is single precision
    int src32, out32;
    unsigned hchi32, hg32;
    // state-vector shards (stage_d2_taylor_kernel<..., SHARD = true>): the top shard_bits qubits of the global index
    // select the shard, every other operand is this shard's slice of 2^(N - shard_bits) amplitudes.  peer[q] = chi_k
    // of shard (shard ^ 1 << q): a flip of shard bit q leaves the local index unchanged
    const c2* peer[PB200_MAX_SHARD_BITS];
    int shard_bits, shard;
    // complex drive on the step (stage kernels with CPLX = true): omega_j = om_j + i omi_j, so the drive part of H_j
    // chi is om_j G + omi_j G', G' = X' chi the gather with factors i unit (X' = sum_k (i unit |to><from|_k + h.c.)).
    // Both come from the same partner loads: G = P + Q, G' = i (P - Q) with P, Q the to-side and from-side sums.
    c2* g2_out;        // G'_k (nullptr: nobody reads it later)
    double om0i;
    const c2* hg2[PB200_TAYLOR_PMAX];    // G'_{k-j}   (nullptr when omi_j = 0)
    double homi[PB200_TAYLOR_PMAX];
    // master equation (stage kernels with DISS = true): the state is vec(rho) of n_pair atoms, s = (r << n_pair) | c,
    // and (k+1) chi_{k+1} = h (-i H chi_k + D chi_k - i sum_j H_j chi_{k-j}): the dissipator D is static, so it acts on
    // chi_k alone and never enters G_k.  Every atom carries the same 4 x 4 generator Gen on its (row bit, column bit)
    // pair, with no entry that flips exactly one of the two bits:
    //   diagonal   dw[0] + dw[1] popc(r) + dw[2] popc(c) + dw[3] popc(r & c)
    //   both-flip  df[i] chi[s ^ pair bits], i = 2 row bit + column bit of s, df[i] = Gen[i][3 - i]
    c2 dw[4], df[4];
    int n_pair;        // 0: no dissipator
    int diss_flip;     // 0: every df is zero (dephasing): no partner loads
};

// epilogue of one amplitude block: everything after the partner sums.  idx is the index inside the trajectory, voff
// the trajectory's offset.  The own-element operands are loaded H amplitudes at a time.  SHARD: idx is local, the
// excitation count is that of the global index (the shard index holds its top bits).  The local detuning of amplitude
// r is either `off[r]` = sum_k c_k [digit_k == from] of the one shape (0 for uniform drives), or, with several shapes,
// a functor off(r, J) = sum_s m_{s,J} sum_k c_{k,s} [digit_k == from] with the shapes' order-0 coefficients (J = 0)
// or those of history term J - 1.
// dint(r) is the interaction diagonal of amplitude r.  v is consumed: with acc_add_h, chi_{k-1} is added into it once the
// diagonal term no longer needs it, so the accumulator update reads no extra operand.
// CPLX: (qx, qy) is G' of the complex-drive step.  DISS: (ex, ey) = i D chi_k, added to the sum that -i h / (k+1) scales.
// HIST32: a history operand may be single precision (TaylorArgs::hchi32, hg32); OUT32: chi_{k+1} and G_k are stored so.
template <int R, int H = (R >= 4) ? R / 2 : R, bool SHARD = false, bool CPLX = false, bool DISS = false,
          bool HIST32 = false, bool OUT32 = false, class Off, class Dint>
__device__ __forceinline__ void taylor_epilogue(const TaylorArgs& a, const long long (&idx)[R], c2 (&v)[R],
                                                const double (&gx)[R], const double (&gy)[R], const Off& off,
                                                long long voff, const Dint& dint,
                                                const double* qx = nullptr, const double* qy = nullptr,
                                                const double* ex = nullptr, const double* ey = nullptr) {
    constexpr bool SHAPES = !std::is_array<Off>::value;
    const int nb = a.geo.n_bits;
    const int ones_hi = SHARD ? __popc(a.shard) : 0;
#pragma unroll
    for (int h0 = 0; h0 < R; h0 += H) {
        double sx[H], sy[H], cn[H];
        {
            double dv[H];
#pragma unroll
            for (int r = 0; r < H; ++r) dv[r] = dint(h0 + r);
#pragma unroll
            for (int r = 0; r < H; ++r) {
                const int ones = __popcll((unsigned long long)idx[h0 + r]) + ones_hi;
                cn[r] = (double)(a.from_is_one ? ones : (nb - ones));
                double diag;
                if constexpr (SHAPES) diag = fma(-a.th0, cn[r], dv[r] - a.gam0 - off(h0 + r, 0));
                else diag = fma(-a.th0, cn[r], fma(-a.m0[0], off[h0 + r], dv[r] - a.gam0));
                sx[r] = fma(diag, v[h0 + r].x, a.om0 * gx[h0 + r]);
                sy[r] = fma(diag, v[h0 + r].y, a.om0 * gy[h0 + r]);
                if constexpr (CPLX) { sx[r] = fma(a.om0i, qx[h0 + r], sx[r]); sy[r] = fma(a.om0i, qy[h0 + r], sy[r]); }
                if constexpr (DISS) { sx[r] += ex[h0 + r]; sy[r] += ey[h0 + r]; }
            }
        }
        for (int j = 0; j < a.nh; ++j) {
            if (a.hchi[j]) {
                c2 c[H];
                if (HIST32 && ((a.hchi32 >> j) & 1)) {
                    const float2* src = reinterpret_cast<const float2*>(a.hchi[j]) + voff;
#pragma unroll
                    for (int r = 0; r < H; ++r) c[r] = ld_own(src + idx[h0 + r]);
                } else {
#pragma unroll
                    for (int r = 0; r < H; ++r) c[r] = ld_own(a.hchi[j] + voff + idx[h0 + r]);
                }
#pragma unroll
                for (int r = 0; r < H; ++r) {
                    double d;
                    if constexpr (SHAPES) d = -fma(a.hth[j], cn[r], a.hgam[j] + off(h0 + r, j + 1));
                    else d = -fma(a.hth[j], cn[r], fma(a.hm[0][j], off[h0 + r], a.hgam[j]));
                    sx[r] = fma(d, c[r].x, sx[r]); sy[r] = fma(d, c[r].y, sy[r]);
                    if (j == 0 && a.acc_add_h) v[h0 + r] = cadd(v[h0 + r], c[r]);
                }
            }
            if (a.hg[j]) {
                c2 c[H];
                if (HIST32 && ((a.hg32 >> j) & 1)) {
                    const float2* src = reinterpret_cast<const float2*>(a.hg[j]) + voff;
#pragma unroll
                    for (int r = 0; r < H; ++r) c[r] = ld_own(src + idx[h0 + r]);
                } else {
#pragma unroll
                    for (int r = 0; r < H; ++r) c[r] = ld_own(a.hg[j] + voff + idx[h0 + r]);
                }
#pragma unroll
                for (int r = 0; r < H; ++r) { sx[r] = fma(a.hom[j], c[r].x, sx[r]); sy[r] = fma(a.hom[j], c[r].y, sy[r]); }
            }
            if constexpr (CPLX) {
                if (a.hg2[j]) {
                    c2 c[H];
#pragma unroll
                    for (int r = 0; r < H; ++r) c[r] = ld_own(a.hg2[j] + voff + idx[h0 + r]);
#pragma unroll
                    for (int r = 0; r < H; ++r) { sx[r] = fma(a.homi[j], c[r].x, sx[r]); sy[r] = fma(a.homi[j], c[r].y, sy[r]); }
                }
            }
        }
        c2 res[H];
#pragma unroll
        for (int r = 0; r < H; ++r) {
            res[r] = {a.scale.x * sx[r] - a.scale.y * sy[r], a.scale.x * sy[r] + a.scale.y * sx[r]};
            // chi_{k+1} is the next order's gather source: kept in L2 ahead of the ring buffers read once per order
            // (C2 on H100: the ring is twice the 50 MB L2; 42.9 against 44.1 us per order, DESIGN.md section 8)
            if constexpr (OUT32) {
                st_c2_evict_last(reinterpret_cast<float2*>(a.out) + voff + idx[h0 + r], res[r]);
                if (a.g_out) st_c2(reinterpret_cast<float2*>(a.g_out) + voff + idx[h0 + r], c2{gx[h0 + r], gy[h0 + r]});
            } else {
                st_c2_evict_last(a.out + voff + idx[h0 + r], res[r]);
                if (a.g_out) st_c2(a.g_out + voff + idx[h0 + r], c2{gx[h0 + r], gy[h0 + r]});
            }
            if constexpr (CPLX) { if (a.g2_out) st_c2(a.g2_out + voff + idx[h0 + r], c2{qx[h0 + r], qy[h0 + r]}); }
        }
        if (a.acc_on) {
            c2 ac[H];
#pragma unroll
            for (int r = 0; r < H; ++r) ac[r] = a.acc_read ? ld_own(a.acc + voff + idx[h0 + r]) : c2{0.0, 0.0};
#pragma unroll
            for (int r = 0; r < H; ++r) {
                c2 s = cadd(ac[r], res[r]);
                if (a.acc_add_v) s = cadd(s, v[h0 + r]);
                st_c2(a.acc + voff + idx[h0 + r], cmul(a.acc_mul, s));
            }
        }
    }
}

// master equation (TaylorArgs::dw): the diagonal of the dissipator at s times chi_k[s]
__device__ __forceinline__ c2 taylor_diss_diag(const TaylorArgs& a, long long s, c2 v) {
    const unsigned long long c = (unsigned long long)s & ((1ULL << a.n_pair) - 1), r = (unsigned long long)s >> a.n_pair;
    const double nr = (double)__popcll(r), nc = (double)__popcll(c), nrc = (double)__popcll(r & c);
    const double wx = fma(a.dw[3].x, nrc, fma(a.dw[2].x, nc, fma(a.dw[1].x, nr, a.dw[0].x)));
    const double wy = fma(a.dw[3].y, nrc, fma(a.dw[2].y, nc, fma(a.dw[1].y, nr, a.dw[0].y)));
    return {wx * v.x - wy * v.y, wx * v.y + wy * v.x};
}

// master equation (TaylorArgs::df): (dx, dy) += the both-flip entry of the pair (row bit pr, column bit pc) at s times
// the partner chi_k[s ^ 2^pr ^ 2^pc] = pv
__device__ __forceinline__ void taylor_diss_flip(const TaylorArgs& a, long long s, int pr, int pc, double2 pv, double& dx,
                                                 double& dy) {
    const c2 f = a.df[(int)((((s >> pr) & 1) << 1) | ((s >> pc) & 1))];
    dx = fma(f.x, pv.x, dx); dx = fma(-f.y, pv.y, dx);
    dy = fma(f.x, pv.y, dy); dy = fma(f.y, pv.x, dy);
}

// ---- interaction diagonal inside the tiled Taylor stage ------------------------------------------------------------
// Dint[s] = sum_{p<q} W_pq [bit p = ryd_bit][bit q = ryd_bit], W_pq = U of the atoms at bit positions p and q
// (TaylorArgs::cpl), factorised along the stage's index
// layout idx = base + tid + m NT (m = c RC + r, RB register bits above the TBITS - RB bits of tid): the bits above the
// tile are fixed per CTA, those of tid per thread, so that
//     Dint = xt[0][tid] + ts[m] + sum_{q : bit q of m = 1} xt[1 + q][tid]
//   ts[m]     = sum over the register bits set in m of (their pairs + their couplings to the set bits above the tile)
//   xt[0]     = the pair sum of the set bits above the tile and in tid   (+ sum_q y_q when ryd_bit = 0)
//   xt[1 + q] = y_q = the couplings of register bit q to the set bits of tid   (negated when ryd_bit = 0: "set" is
//               then bit q = 0, and sum_{q : bit = 0} y_q = sum_q y_q - sum_{q : bit = 1} y_q)
// Shared memory, in doubles: wt[TBITS^2] couplings among the tile bits, wj[TBITS] couplings of each tile bit to the set
// bits above the tile, hh their pair sum, ts[2^RB], xt[RB + 1][NT], then a copy of the N x N matrix.
__host__ __device__ constexpr int taylor_dint_doubles(int tbits, int rb) {
    return tbits * tbits + tbits + 1 + (1 << rb) + (rb + 1) * (1 << (tbits - rb));
}

// fills the shared-memory factors above; ends with this thread's xt written (read back by this thread only).  hi: the
// global index bits above the tile of this CTA (a shard's index included).  Contains __syncthreads.
template <int TBITS, int RB>
__device__ __forceinline__ void taylor_dint_setup(const TaylorArgs& a, long long traj, unsigned long long hi, int tid,
                                                  double* dsm) {
    constexpr int NT = 1 << (TBITS - RB), L0 = TBITS - RB;
    const int nb = a.geo.n_bits;
    double* Ws = dsm + taylor_dint_doubles(TBITS, RB);   // the whole matrix, one coalesced pass
    const double* Wq = a.cpl + traj * a.cpl_stride;
    for (int i = tid; i < nb * nb; i += NT) Ws[i] = __ldg(Wq + i);
    __syncthreads();
    auto W = [&](int p, int q) { return Ws[(nb - 1 - p) * nb + (nb - 1 - q)]; };   // atom nb - 1 - p at bit p
    const unsigned long long flip = a.ryd_bit ? 0ULL : ~0ULL;
    const unsigned long long nmask = nb >= 64 ? ~0ULL : (1ULL << nb) - 1;
    const unsigned long long hs = (hi ^ flip) & nmask & ~((1ULL << TBITS) - 1);   // set bits above the tile
    double* wt = dsm;
    double* wj = wt + TBITS * TBITS;
    double* hh = wj + TBITS;
    double* ts = hh + 1;
    double* xt = ts + (1 << RB);
    for (int i = tid; i < TBITS * TBITS; i += NT) wt[i] = W(i / TBITS, i % TBITS);
    if (tid < TBITS) {
        double s = 0.0;
        for (unsigned long long m = hs; m; m &= m - 1) s += W(__ffsll((long long)m) - 1, tid);
        wj[tid] = s;
    } else if (tid >= 32 && tid < 32 + (1 << RB)) {
        const int m = tid - 32;
        const unsigned ms = ((unsigned)m ^ (unsigned)flip) & ((1u << RB) - 1);
        double s = 0.0;
        for (int q = 0; q < RB; ++q) {
            if (!((ms >> q) & 1)) continue;
            for (unsigned long long h = hs; h; h &= h - 1) s += W(L0 + q, __ffsll((long long)h) - 1);
            for (int q2 = q + 1; q2 < RB; ++q2) if ((ms >> q2) & 1) s += W(L0 + q, L0 + q2);
        }
        ts[m] = s;
    } else if (tid >= 64 && tid < 96) {
        double s = 0.0;
        for (int p = TBITS + (tid - 64); p < nb; p += 32) {
            if (!((hs >> p) & 1)) continue;
            for (unsigned long long h = hs & ~((2ULL << p) - 1); h; h &= h - 1) s += W(p, __ffsll((long long)h) - 1);
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (tid == 64) hh[0] = s;
    }
    __syncthreads();
    const unsigned tb = ((unsigned)tid ^ (unsigned)flip) & (NT - 1);   // set bits of tid
    double ct = hh[0];
    double y[RB];
#pragma unroll
    for (int q = 0; q < RB; ++q) y[q] = 0.0;
#pragma unroll 1
    for (int i = 0; i < L0; ++i) {
        const bool bi = (tb >> i) & 1;
        ct += bi ? wj[i] : 0.0;
        for (int j = i + 1; j < L0; ++j) ct += (bi && ((tb >> j) & 1)) ? wt[i * TBITS + j] : 0.0;
#pragma unroll
        for (int q = 0; q < RB; ++q) y[q] += bi ? wt[i * TBITS + L0 + q] : 0.0;
    }
#pragma unroll
    for (int q = 0; q < RB; ++q) {
        if (!a.ryd_bit) { ct += y[q]; y[q] = -y[q]; }
        xt[(q + 1) * NT + tid] = y[q];
    }
    xt[tid] = ct;
}

// UNIFORM: one drive coefficient for every qubit and a single state (C2, C5); otherwise per-(trajectory, qubit) static
// factors from `table`, blockIdx.y = trajectory (C4: doppler + amplitude noise batches).
// The tile is the TBITS low bits of the index (taylor_geometry), the bits above it are coalesced partner loads.  A thread
// owns R = 2^RB amplitudes (tile index t = tid + r*NT) and works through them in chunks of 8: chunk c is the sub-tile
// whose top RB - 3 tile bits equal c, where the register-blocked gather of rb_tile_gather applies, and a flip of a chunk
// bit is one more LDS.128 from the other chunk's sub-tile.  Only one chunk's partner sums are live at a time, which is
// what lets 16 amplitudes per thread fit in 128 registers; the first chunk's partner loads overlap the tile copy.
// SHARD (uniform drives): the launch works on one shard of the state (TaylorArgs::peer); a flip of shard bit q is one
// more coalesced load from the peer's chi_k at the same local index, issued with the other out-of-tile partners.
// NS: detuning shapes with per-bit weights.  0 (uniform) and 1 (batch) read the one-shape table of d2_table_stride;
// PB200_TAYLOR_SMAX reads taylor_table_stride(N, PB200_TAYLOR_SMAX), with a uniform drive too (detuning maps).  Only
// the combinations sum_s m_{s,J} off_s of the order's coefficients enter the diagonal, so they are formed once per
// launch in shared memory (per thread for the bits of base + tid, per register-bit pattern for the rest) and an
// amplitude reads two of them per history term instead of holding S offsets in registers.
// CPLX: the drive's phase moves inside the step (TaylorArgs::om0i, hg2, g2_out): the per-bit table gather also forms
// the signed sum P - Q of the same partner loads, i.e. G' as well as G.  The two sums of a chunk do not fit in 128
// registers; these launches use fewer threads with more chunks each (kTaylorCplxRegBits) and one CTA's worth of
// registers per SM.
// DISS: the master equation on vec(rho) (TaylorArgs::dw, df; the batch gather, whose per-bit table carries the column
// drive -conj(omega)).  The dissipator sum of a chunk is a second accumulator, which does not fit in 128 registers
// either: the same launch shape as CPLX.  A pair whose row bit lies in the tile reads its both-flip partner from shared
// memory, one above the tile costs one more coalesced load per atom.  DISS with SHARD: vec(rho) split by its top row
// bits (one trajectory); the per-bit table's entries of the shard bits drive the peer loads, and a pair whose row bit
// is a shard bit reads its both-flip partner from that peer.
// CPLX with DISS: vec(rho) under a drive whose phase moves.  Row bit k sees unit omega, column bit k -conj(unit)
// conj(omega) (the table holds f = unit on row bits and -conj(unit) on column bits), so the drive part of H_j is
// om_j G + omi_j G' where G' is the CPLX signed sum with the sign of every column bit (position < n_pair) negated: the
// column's y-factor is i conj(unit) = -i f.  The dissipator acts on chi_k alone, as without CPLX.  One state only.
// SRC32 / OUT32: the tail orders of a step (TaylorStep::k_lo), uniform drives of one state (or its shards) only.  chi_k (tile and
// partners) is read as float2, chi_{k+1} and G_k are stored as float2; the arithmetic, the partner sums and the
// accumulator stay fp64.  The single-precision tile fills the first 64 KiB of the tile's 128.
template <bool UNIFORM, bool REAL_G, int TBITS, int RB, bool SHARD = false, int NS = (UNIFORM ? 0 : 1), bool CPLX = false,
          bool DISS = false, bool SRC32 = false, bool OUT32 = false>
__global__ void __launch_bounds__(1 << (TBITS - RB),
                                  (CPLX || DISS) ? 1 : (65536 / ((1 << (TBITS - RB)) * (RB >= 3 ? 128 : 64))))
stage_d2_taylor_kernel(const __grid_constant__ TaylorArgs a) {
    static_assert(RB >= 3, "chunks of 8 amplitudes per thread");
    static_assert(UNIFORM || !SHARD || DISS, "shards carry one state with a uniform drive, or one density matrix");
    static_assert(NS == (UNIFORM ? 0 : 1) || NS == PB200_TAYLOR_SMAX, "one-shape table, or PB200_TAYLOR_SMAX shapes");
    static_assert(!CPLX || !REAL_G, "a complex drive gathers through the per-bit table");
    static_assert(!DISS || (!UNIFORM && !(CPLX && SHARD)),
                  "a density matrix runs the batch gather; a moving phase on whole density matrices only");
    static_assert(!(SRC32 || OUT32) || (UNIFORM && NS == 0 && !CPLX && !DISS),
                  "single-precision orders: one state, a uniform drive of one phase");
    using TT = std::conditional_t<SRC32, float2, c2>;   // element of chi_k
    constexpr bool SHAPES = NS == PB200_TAYLOR_SMAX;
    constexpr int NT = 1 << (TBITS - RB);
    constexpr int TSIZE = 1 << TBITS;
    constexpr int RC = 8;                   // amplitudes per chunk
    constexpr int CB = RB - 3;              // chunk bits: the top CB tile bits
    constexpr int STB = TBITS - CB;         // bits of a chunk's sub-tile
    // complex per-bit drive factors from the shared-memory table: the per-qubit factors, or the unit of a uniform
    // drive of non-zero phase (G = sum_k (unit |to><from|_k + h.c.): one complex factor per partner and two
    // accumulators per amplitude instead of the P and Q sums)
    constexpr bool TAB = !(UNIFORM && REAL_G);
    constexpr bool COLSIGN = CPLX && DISS;   // the signed sums change sign on the column bits of vec(rho)
    extern __shared__ __align__(128) unsigned char smem_raw[];
    TT* tile = reinterpret_cast<TT*>(smem_raw);
    __shared__ __align__(8) uint64_t mbar;
    const PassGeom& g = a.geo;
    const int tid = threadIdx.x;
    const long long traj = UNIFORM ? 0 : (long long)blockIdx.y;
    const long long voff = traj * a.D;
    const long long base = (long long)blockIdx.x << TBITS;
    const TT* vsrc = reinterpret_cast<const TT*>(a.v) + voff;

    if (tid == 0) mbar_init(&mbar, 1);
    __syncthreads();
    double* dsm = reinterpret_cast<double*>(smem_raw + (size_t)TSIZE * sizeof(c2));   // taylor_dint_setup
    const double* ts = dsm + TBITS * TBITS + TBITS + 1;
    const double* xt = ts + (1 << RB);
    double* tab = dsm + taylor_dint_doubles(TBITS, RB) + g.n_bits * g.n_bits;
    // the interaction's factors depend on the plan alone: formed before the wait on the previous order, so that they
    // overlap its tail (behind the first chunk's partner loads, the setup's registers would spill)
    if (a.cpl)
        taylor_dint_setup<TBITS, RB>(
            a, traj, (unsigned long long)base | (SHARD ? (unsigned long long)a.shard << (g.n_bits - a.shard_bits) : 0ULL),
            tid, dsm);
    pdl_wait();
    pdl_launch_dependents();
    if (tid == 0) {
        mbar_arrive_expect_tx(&mbar, (uint32_t)(TSIZE * sizeof(TT)));
        tma_load_1d(tile, vsrc + base, (uint32_t)(TSIZE * sizeof(TT)), &mbar);
    }
    // SHAPES, for J = 0 (order-0 coefficients m0) and J = 1 + history j (hm[s][j]) up to nh, behind the per-bit table:
    //   bl[J][i]   = sum_s m_{s,J} x (shape s's weights of the register bits i, relative to i = 0), the same for all
    //   at[J][tid] = sum_s m_{s,J} x (shape s's weights of the bits of base + tid, shard bits included)
    // so that the local detuning of amplitude (c RC + r) in history J is at[J][tid] + bl[J][c RC + r]
    double* bl = tab + (SHAPES ? taylor_table_stride(g.n_bits, NS) : 0);
    double* at = bl + ((PB200_TAYLOR_PMAX + 1) << RB);
    auto shape_coef = [&](int J, int s) { return J == 0 ? a.m0[s] : a.hm[s][J - 1]; };
    if (TAB || SHAPES) {   // the table is written behind the tile copy
        if (UNIFORM && !SHAPES) {
            for (int i = tid; i < 2 * g.n_bits; i += NT) tab[i] = (i & 1) ? a.unit.y : a.unit.x;
        } else {
            const int stride = SHAPES ? taylor_table_stride(g.n_bits, NS) : d2_table_stride(g.n_bits);
            const double* src = a.table + traj * stride;
            for (int i = tid; i < stride; i += NT) tab[i] = src[i];
            if (SHAPES) {
                for (int i = tid; i < ((a.nh + 1) << RB); i += NT) {
                    const int J = i >> RB;
                    double acc = 0.0;
                    for (int s = 0; s < NS; ++s) {
                        const double* w = src + 2 * g.n_bits + s * g.n_bits + (TBITS - RB);
                        double l = 0.0;
                        for (int q = 0; q < RB; ++q) {
                            const int bit = (i >> q) & 1;
                            l += ((bit == a.from_is_one) ? w[q] : 0.0) - ((0 == a.from_is_one) ? w[q] : 0.0);
                        }
                        acc = fma(shape_coef(J, s), l, acc);
                    }
                    bl[i] = acc;
                }
            }
        }
        __syncthreads();
    }
    const int to_bit = a.to_bit;
    const int nb = g.n_bits;
    // static per-qubit detuning weights: sum over (bits of base) + (bits of tid) + (register bits)
    double common = 0.0;
    if (!UNIFORM && !SHAPES) {   // a shard's global bits N - shard_bits + q are the bits of the shard index
        for (int p = 0; p < nb; ++p) {
            int bit = (int)(((base + tid) >> p) & 1);
            if (SHARD && p >= nb - a.shard_bits) bit = (a.shard >> (p - (nb - a.shard_bits))) & 1;
            common += (bit == a.from_is_one) ? tab[2 * nb + p] : 0.0;
        }
    }
    if (SHAPES) {   // a shard's global bits N - shard_bits + q are the bits of the shard index
        double cs[NS > 0 ? NS : 1];
#pragma unroll
        for (int s = 0; s < NS; ++s) cs[s] = 0.0;
        for (int p = 0; p < nb; ++p) {
            int bit = (int)(((base + tid) >> p) & 1);
            if (SHARD && p >= nb - a.shard_bits) bit = (a.shard >> (p - (nb - a.shard_bits))) & 1;
            if (bit == a.from_is_one) {
#pragma unroll
                for (int s = 0; s < NS; ++s) cs[s] += tab[2 * nb + s * nb + p];
            }
        }
        for (int J = 0; J <= a.nh; ++J) {
            double acc = 0.0;
#pragma unroll
            for (int s = 0; s < NS; ++s) acc = fma(shape_coef(J, s), cs[s], acc);
            at[J * NT + tid] = acc;   // read by this thread only
        }
    }
#pragma unroll 1
    for (int c = 0; c < (1 << CB); ++c) {
        const long long i0 = base + tid + c * RC * NT;   // index of the chunk's first amplitude; the r-th is i0 + r*NT
        double pr[RC], pi[RC];
        double dr[RC], di[RC];   // CPLX: signed sums P - Q
#pragma unroll
        for (int r = 0; r < RC; ++r) { pr[r] = 0.0; pi[r] = 0.0; dr[r] = 0.0; di[r] = 0.0; }
        // partners across the bits outside the tile: coalesced loads (for the first chunk, while the tile is in flight)
        for (unsigned long long m = g.extra_mask; m; m &= m - 1) {
            const int p = __ffsll((long long)m) - 1;
            const int bit = (int)((base >> p) & 1);
            double gx = 0.0, gy = 0.0;
            if (TAB) { gx = tab[2 * p]; gy = (bit == to_bit) ? tab[2 * p + 1] : -tab[2 * p + 1]; }
            const TT* src = vsrc + (i0 ^ (1LL << p));
            const bool col = COLSIGN && p < a.n_pair;
            double2 raw[RC];
#pragma unroll
            for (int r = 0; r < RC; ++r) raw[r] = ld_partner(src + r * NT);
#pragma unroll
            for (int r = 0; r < RC; ++r) {
                if constexpr (CPLX) {
                    taylor_signed_add(gx, gy, ((bit == to_bit) != col) ? 1.0 : -1.0, raw[r].x, raw[r].y, pr[r], pi[r], dr[r],
                                      di[r]);
                } else if (!TAB) {
                    pr[r] += raw[r].x; pi[r] += raw[r].y;
                } else {
                    pr[r] = fma(gx, raw[r].x, pr[r]); pr[r] = fma(-gy, raw[r].y, pr[r]);
                    pi[r] = fma(gx, raw[r].y, pi[r]); pi[r] = fma(gy, raw[r].x, pi[r]);
                }
            }
        }
        if (SHARD) {
            // partners across the shard bits (global bits N - shard_bits + q): same local index in the peer's slice,
            // the sign of the drive term from the global bit value, i.e. the shard index
            for (int q = 0; q < a.shard_bits; ++q) {
                const int bit = (a.shard >> q) & 1;
                double gx = 0.0, gy = 0.0;
                if (TAB) {
                    const int p = nb - a.shard_bits + q;
                    gx = tab[2 * p]; gy = (bit == to_bit) ? tab[2 * p + 1] : -tab[2 * p + 1];
                }
                const TT* src = reinterpret_cast<const TT*>(a.peer[q]) + i0;
                double2 raw[RC];
#pragma unroll
                for (int r = 0; r < RC; ++r) {
                    if constexpr (SRC32) raw[r] = make_double2((double)src[r * NT].x, (double)src[r * NT].y);
                    else raw[r] = *reinterpret_cast<const double2*>(src + r * NT);
                }
#pragma unroll
                for (int r = 0; r < RC; ++r) {
                    if constexpr (CPLX) {
                        taylor_signed_add(gx, gy, bit == to_bit ? 1.0 : -1.0, raw[r].x, raw[r].y, pr[r], pi[r], dr[r], di[r]);
                    } else if (!TAB) {
                        pr[r] += raw[r].x; pi[r] += raw[r].y;
                    } else {
                        pr[r] = fma(gx, raw[r].x, pr[r]); pr[r] = fma(-gy, raw[r].y, pr[r]);
                        pi[r] = fma(gx, raw[r].y, pi[r]); pi[r] = fma(gy, raw[r].x, pi[r]);
                    }
                }
            }
        }
        if (c == 0) mbar_wait(&mbar, 0);
        auto dint = [&](int r) {
            if (!a.cpl) return 0.0;
            const int m = c * RC + r;
            double d = ts[m] + xt[tid];
#pragma unroll
            for (int q = 0; q < RB; ++q)
                if ((m >> q) & 1) d += xt[(q + 1) * NT + tid];
            return d;
        };
        const TT* sub = tile + (c << STB);
        c2 v[RC];
        double qd[RC];   // the Q sums of rb_tile_gather: not used by the two instantiations below
#pragma unroll
        for (int r = 0; r < RC; ++r) v[r] = tile_c2(sub[tid + r * NT]);
        if constexpr (CPLX)
            rb_tile_gather<false, false, STB, 3, true, COLSIGN>(g, sub, tab, tid, to_bit, 0, false, v, pr, pi, dr, di, a.n_pair);
        else rb_tile_gather<!TAB, !TAB, STB, 3>(g, sub, tab, tid, to_bit, 0, false, v, pr, pi, qd, qd);
#pragma unroll
        for (int q = 0; q < CB; ++q) {   // flips of the chunk bits
            const int p = STB + q;
            const int bit = (c >> q) & 1;
            const bool col = COLSIGN && p < a.n_pair;
            double gx = 0.0, gy = 0.0;
            if (TAB) { gx = tab[2 * p]; gy = (bit == to_bit) ? tab[2 * p + 1] : -tab[2 * p + 1]; }
            const TT* other = tile + ((c ^ (1 << q)) << STB);
#pragma unroll
            for (int r = 0; r < RC; ++r) {
                const c2 pv = tile_c2(other[tid + r * NT]);
                if constexpr (CPLX) {
                    taylor_signed_add(gx, gy, ((bit == to_bit) != col) ? 1.0 : -1.0, pv.x, pv.y, pr[r], pi[r], dr[r], di[r]);
                } else if (!TAB) {
                    pr[r] += pv.x; pi[r] += pv.y;
                } else {
                    pr[r] = fma(gx, pv.x, pr[r]); pr[r] = fma(-gy, pv.y, pr[r]);
                    pi[r] = fma(gx, pv.y, pi[r]); pi[r] = fma(gy, pv.x, pi[r]);
                }
            }
        }
        double off[RC];
        long long idx[RC];
#pragma unroll
        for (int r = 0; r < RC; ++r) {
            idx[r] = i0 + r * NT;
            if (!TAB) { pr[r] *= a.unit.x; pi[r] *= a.unit.x; }   // G = ux P for a real unit
            double acc = common;
            if (!UNIFORM && !SHAPES) {
#pragma unroll
                for (int q = 0; q < RB; ++q) {
                    const double th = tab[2 * nb + TBITS - RB + q];
                    const int bit = ((c * RC + r) >> q) & 1;   // `base + tid` has these bits at 0
                    acc += ((bit == a.from_is_one) ? th : 0.0) - ((0 == a.from_is_one) ? th : 0.0);
                }
            }
            off[r] = acc;
        }
        double ex[RC], ey[RC];   // DISS: i D chi_k
        if constexpr (DISS) {
            // SHARD: the dissipator reads the row and column bits of the global index (the shard index holds the top
            // row bits)
            const long long goff = SHARD ? (long long)a.shard << (nb - a.shard_bits) : 0LL;
            double dx[RC], dy[RC];
#pragma unroll
            for (int r = 0; r < RC; ++r) {
                const c2 w = taylor_diss_diag(a, goff | idx[r], v[r]);
                dx[r] = w.x; dy[r] = w.y;
            }
            if (a.diss_flip) {
                const int tpos = tid + (c << STB);   // tile position of the chunk's first amplitude
                for (int pc = 0; pc < a.n_pair; ++pc) {
                    const int pr = pc + a.n_pair;
                    const long long mask = (1LL << pr) | (1LL << pc);
                    double2 pv[RC];
                    if (pr < TBITS) {
#pragma unroll
                        for (int r = 0; r < RC; ++r) {
                            const c2 t = tile_c2(tile[(tpos + r * NT) ^ (int)mask]);
                            pv[r] = make_double2(t.x, t.y);
                        }
                    } else if (SHARD && pr >= nb - a.shard_bits) {
                        // the row bit is shard bit q: the partner is the peer's, at the local index with the column
                        // bit flipped (the column bits are all local)
                        const TT* src = reinterpret_cast<const TT*>(a.peer[pr - (nb - a.shard_bits)]);
#pragma unroll
                        for (int r = 0; r < RC; ++r) pv[r] = ld_partner(src + (idx[r] ^ (1LL << pc)));
                    } else {
#pragma unroll
                        for (int r = 0; r < RC; ++r) pv[r] = ld_partner(vsrc + (idx[r] ^ mask));
                    }
#pragma unroll
                    for (int r = 0; r < RC; ++r) taylor_diss_flip(a, goff | idx[r], pr, pc, pv[r], dx[r], dy[r]);
                }
            }
#pragma unroll
            for (int r = 0; r < RC; ++r) { ex[r] = -dy[r]; ey[r] = dx[r]; }
        }
        // per-qubit factors (off != 0) leave the registers for 2 amplitudes' operands at a time, not 4
        if constexpr (CPLX) {
            double qx[RC], qy[RC];   // G' = i (P - Q)
#pragma unroll
            for (int r = 0; r < RC; ++r) { qx[r] = -di[r]; qy[r] = dr[r]; }
            if constexpr (SHAPES) {
                const double* lc = bl + c * RC;
                const double* lt = at + tid;
                taylor_epilogue<RC, RC / 4, SHARD, true, DISS>(
                    a, idx, v, pr, pi, [&](int r, int J) { return lt[J * NT] + lc[(J << RB) + r]; }, voff, dint, qx, qy,
                    ex, ey);
            } else {
                taylor_epilogue<RC, RC / 4, SHARD, true, DISS>(a, idx, v, pr, pi, off, voff, dint, qx, qy, ex, ey);
            }
        } else if constexpr (SHAPES) {
            const double* lc = bl + c * RC;
            const double* lt = at + tid;
            taylor_epilogue<RC, RC / 4, SHARD, false, DISS>(
                a, idx, v, pr, pi, [&](int r, int J) { return lt[J * NT] + lc[(J << RB) + r]; }, voff, dint, nullptr,
                nullptr, ex, ey);
        } else {
            taylor_epilogue<RC, UNIFORM ? RC / 2 : RC / 4, SHARD, false, DISS, SRC32, OUT32>(a, idx, v, pr, pi, off, voff,
                                                                                           dint, nullptr, nullptr, ex, ey);
        }
    }
}

// any register size (N < 13 in particular): one thread per amplitude, partners through global loads.  CPLX: the
// complex-drive step, G' = i (P - Q) as well (stage_d2_taylor_kernel).  DISS: the master equation on vec(rho), the
// both-flip partners through global loads too.  Both: the signed sum changes sign on the column bits.
template <bool CPLX = false, bool DISS = false>
__global__ void __launch_bounds__(256) stage_d2_taylor_small_kernel(const __grid_constant__ TaylorArgs a) {
    const long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= a.D) return;
    const int nb = a.geo.n_bits;
    const long long traj = blockIdx.y;
    const long long voff = traj * a.D;
    const int ns = a.tab_shapes ? a.tab_shapes : 1;
    const double* tab = a.table ? a.table + traj * (a.tab_shapes ? taylor_table_stride(nb, ns) : d2_table_stride(nb)) : nullptr;
    double gxs = 0.0, gys = 0.0, offv[PB200_TAYLOR_SMAX];
    double q2x = 0.0, q2y = 0.0;   // CPLX: G'
#pragma unroll
    for (int q = 0; q < PB200_TAYLOR_SMAX; ++q) offv[q] = 0.0;
    if (tab) {
        double dx = 0.0, dy = 0.0;
        for (int p = 0; p < nb; ++p) {
            const double2 raw = __ldg(reinterpret_cast<const double2*>(a.v + voff + (s ^ (1LL << p))));
            const int bit = (int)((s >> p) & 1);
            const double gx = tab[2 * p], gy = (bit == a.to_bit) ? tab[2 * p + 1] : -tab[2 * p + 1];
            if constexpr (CPLX) {
                const bool col = DISS && p < a.n_pair;   // vec(rho): the column bits' signed sum changes sign
                taylor_signed_add(gx, gy, ((bit == a.to_bit) != col) ? 1.0 : -1.0, raw.x, raw.y, gxs, gys, dx, dy);
            } else {
                gxs = fma(gx, raw.x, gxs); gxs = fma(-gy, raw.y, gxs);
                gys = fma(gx, raw.y, gys); gys = fma(gy, raw.x, gys);
            }
            if (bit == a.from_is_one) {
#pragma unroll
                for (int q = 0; q < PB200_TAYLOR_SMAX; ++q)
                    if (q < ns) offv[q] += tab[2 * nb + q * nb + p];
            }
        }
        q2x = -dy; q2y = dx;
    } else {
        double pr = 0.0, pi = 0.0, qr = 0.0, qi = 0.0;
        for (int p = 0; p < nb; ++p) {
            const double2 raw = __ldg(reinterpret_cast<const double2*>(a.v + voff + (s ^ (1LL << p))));
            const double sg = ((int)((s >> p) & 1) == a.to_bit) ? 1.0 : -1.0;
            pr += raw.x; pi += raw.y; qr = fma(sg, raw.x, qr); qi = fma(sg, raw.y, qi);
        }
        gxs = fma(-a.unit.y, qi, a.unit.x * pr);
        gys = fma(a.unit.y, qr, a.unit.x * pi);
        // P - Q = ux Q + i uy P in these sums (Q here is the signed sum)
        q2x = -fma(a.unit.x, qi, a.unit.y * pr);
        q2y = fma(a.unit.x, qr, -a.unit.y * pi);
    }
    const long long idx[1] = {s};
    const double2 own = __ldg(reinterpret_cast<const double2*>(a.v + voff + s));
    c2 v[1] = {{own.x, own.y}};
    const double gx[1] = {gxs}, gy[1] = {gys}, offv1[1] = {offv[0]};
    const double qx[1] = {q2x}, qy[1] = {q2y};
    double ex[1] = {0.0}, ey[1] = {0.0};   // DISS: i D chi_k
    if constexpr (DISS) {
        const c2 w = taylor_diss_diag(a, s, v[0]);
        double dx = w.x, dy = w.y;
        if (a.diss_flip) {
            for (int pc = 0; pc < a.n_pair; ++pc) {
                const int pr = pc + a.n_pair;
                const double2 pv = __ldg(reinterpret_cast<const double2*>(a.v + voff + (s ^ (1LL << pr) ^ (1LL << pc))));
                taylor_diss_flip(a, s, pr, pc, pv, dx, dy);
            }
        }
        ex[0] = -dy; ey[0] = dx;
    }
    auto local = [&](int, int J) {
        double acc = 0.0;
#pragma unroll
        for (int q = 0; q < PB200_TAYLOR_SMAX; ++q) acc = fma(J == 0 ? a.m0[q] : a.hm[q][J - 1], offv[q], acc);
        return acc;
    };
    const double* dsrc = a.dint ? a.dint + traj * a.dint_stride : nullptr;
    auto dint = [&](int) { return dsrc ? __ldcs(dsrc + s) : 0.0; };
    if (a.tab_shapes) taylor_epilogue<1, 1, false, CPLX, DISS>(a, idx, v, gx, gy, local, voff, dint, qx, qy, ex, ey);
    else taylor_epilogue<1, 1, false, CPLX, DISS>(a, idx, v, gx, gy, offv1, voff, dint, qx, qy, ex, ey);
}

// ---- generic-d stage kernel (any dim, several drives; global gathers) -------
// table per (exponential, trajectory):
//   for each drive q: g[q][k] (re,im) per QUDIT k, theta[q][k]; then w, gamma
// per-(exponential, trajectory) table of the generic kernel: per drive q [g (re,im) per qudit | theta per qudit],
// then wc (weight of the SLM-masked part of the interaction, XY mode), w, gamma
__host__ __device__ inline int gen_table_stride(int n, int n_drives) { return n_drives * 3 * n + 3; }

#define PB200_TILED_MAX_HIGH 40
#define PB200_MAX_DRIVES_K 3
struct GenArgs {
    const c2* v; const c2* psi; const c2* b2; c2* out;
    const double* dint; long long dint_stride; long long D;
    int n, dim, n_drives;
    int to[3], from[3];
    StageCoef coef;
    const double* table;  // [B][stride]
    const double* beta_dev;
    // XY mode: exchange couplings U^xy_ij (|u d><d u| + h.c.), [Bx][n*n], weighted by the table's w like Dint
    const double* xy; long long xy_stride; int xy_u, xy_d;
    // XY mode with an SLM mask (hamiltonian.py:399-424): pairs touching a masked qudit (bit k of slm_mask) carry the
    // weight wc = table[stride - 3] instead of w; dint2 = interaction diagonal of those pairs (dint: the others)
    unsigned long long slm_mask; const double* dint2;
    double* dot_acc;   // fused reductions (register-blocked tiled kernel only): acc[traj][0] += Re<lhs, out>, [1] += <out, out>
    LanczosFuse lz;    // fused Lanczos step when lz.vj != nullptr (register-blocked tiled kernel only)
};

__global__ void __launch_bounds__(256) stage_generic_kernel(GenArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* tab = reinterpret_cast<double*>(smem_raw);
    const int stride = gen_table_stride(a.n, a.n_drives);
    const long long traj = blockIdx.y;
    for (int i = threadIdx.x; i < stride; i += blockDim.x) tab[i] = a.table[traj * stride + i];
    __syncthreads();
    double* xys = tab + stride;  // XY couplings of this trajectory, weighted like Dint
    if (a.xy) {
        const double wx = tab[stride - 2], wxc = tab[stride - 3];
        for (int i = threadIdx.x; i < a.n * a.n; i += blockDim.x) {
            const int qi = i / a.n, qj = i - qi * a.n;
            const bool touched = ((a.slm_mask >> qi) | (a.slm_mask >> qj)) & 1ULL;
            xys[i] = a.xy[traj * a.xy_stride + i] * (touched ? wxc : wx);
        }
        __syncthreads();
    }
    const double w = tab[stride - 2], gamma = tab[stride - 1];
    const long long voff = traj * a.D;
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < a.D;
         idx += (long long)gridDim.x * blockDim.x) {
        const c2 vo = a.v[voff + idx];
        double diag = -gamma;
        if (a.dint) diag = fma(w, a.dint[traj * a.dint_stride + idx], diag);
        if (a.dint2) diag = fma(tab[stride - 3], a.dint2[traj * a.dint_stride + idx], diag);
        double rr = 0.0, ri = 0.0;
        long long rem = idx, st = 1;
        for (int k = a.n - 1; k >= 0; --k) {  // qudit k has stride dim^(n-1-k)
            const int digit = (int)(rem % a.dim);
            rem /= a.dim;
            for (int q = 0; q < a.n_drives; ++q) {
                const double* gq = tab + q * 3 * a.n;
                if (digit == a.to[q]) {
                    const c2 pv = a.v[voff + idx + (long long)(a.from[q] - a.to[q]) * st];
                    const double gx = gq[2 * k], gy = gq[2 * k + 1];
                    rr = fma(gx, pv.x, rr); rr = fma(-gy, pv.y, rr);
                    ri = fma(gx, pv.y, ri); ri = fma(gy, pv.x, ri);
                } else if (digit == a.from[q]) {
                    const c2 pv = a.v[voff + idx + (long long)(a.to[q] - a.from[q]) * st];
                    const double gx = gq[2 * k], gy = -gq[2 * k + 1];
                    rr = fma(gx, pv.x, rr); rr = fma(-gy, pv.y, rr);
                    ri = fma(gx, pv.y, ri); ri = fma(gy, pv.x, ri);
                    diag -= gq[2 * a.n + k];
                }
            }
            st *= a.dim;
        }
        if (a.xy) {  // flip-flop partners: every pair (i, j) holding (u, d) or (d, u)  (make_xy_term, :276-294)
            signed char dg[40];
            long long sts[40];
            long long r2 = idx, s2 = 1;
            for (int k = a.n - 1; k >= 0; --k) { dg[k] = (signed char)(r2 % a.dim); r2 /= a.dim; sts[k] = s2; s2 *= a.dim; }
            for (int i = 0; i < a.n; ++i) {
                if (dg[i] != a.xy_u && dg[i] != a.xy_d) continue;
                for (int j = i + 1; j < a.n; ++j) {
                    if ((dg[i] == a.xy_u && dg[j] == a.xy_d) || (dg[i] == a.xy_d && dg[j] == a.xy_u)) {
                        const double u = xys[i * a.n + j];
                        if (u == 0.0) continue;
                        const long long pidx2 = idx + (long long)(dg[j] - dg[i]) * sts[i] + (long long)(dg[i] - dg[j]) * sts[j];
                        const c2 pv = a.v[voff + pidx2];
                        rr = fma(u, pv.x, rr); ri = fma(u, pv.y, ri);
                    }
                }
            }
        }
        c2 gv = {fma(diag, vo.x, rr), fma(diag, vo.y, ri)};
        c2 res = cmul(a.coef.c_g, gv);
        if (a.psi) res = cadd(res, cmul(a.coef.c_psi, a.psi[voff + idx]));
        if (a.b2) res = cadd(res, cmul(a.beta_dev ? c2{-a.beta_dev[traj], 0.0} : a.coef.c_b2, a.b2[voff + idx]));
        st_c2(a.out + voff + idx, res);
    }
}

// ---- tiled stage kernel for d = 3 / 4 (the "all" basis, leakage levels) ---------------------------------------
// Same maths as stage_generic_kernel without the XY exchange term.  A CTA owns the DIM^K amplitudes that share
// their n - K most significant digits (one contiguous run, brought in by ONE TMA bulk copy): partners across the
// K low digits are shared-memory reads selected arithmetically (no divergence: a digit that is neither |to> nor
// |from> of a drive reads itself with a zero coefficient); the high digits are the same for the whole tile, so
// their partners are a short CTA-uniform list of (offset, coefficient) pairs served by coalesced loads.
struct TileExtra { long long off; double gx, gy; };

// ---- register-blocked tiled stage kernel for d = 3 / 4 --------------------------------------------------------
// stage_tiled_kernel is instruction-bound (ncu on C3: 1053 thread instructions per amplitude, issue-active 62 %,
// DRAM 10 %: the digit decomposition, the coefficient selects and the table reads are redone for every amplitude).
// Here a thread owns the R = DIM^RBD amplitudes that differ in the top RBD tile digits and keeps their
// accumulators in registers: digits, selects and coefficients are computed once per (digit, drive) and reused for
// the R amplitudes, exactly as the d = 2 kernel reuses them across its register block.
__host__ __device__ constexpr int ipow_c(int b, int e) { return e <= 0 ? 1 : b * ipow_c(b, e - 1); }

template <int DIM, int K, int RBD>
__global__ void __launch_bounds__(256, 2) stage_multilevel_rb_kernel(GenArgs a) {
    constexpr int R = ipow_c(DIM, RBD);
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ __align__(8) uint64_t mbar;
    __shared__ TileExtra extra[PB200_MAX_DRIVES_K * PB200_TILED_MAX_HIGH];
    __shared__ int n_extra;
    __shared__ double diag_high;

    const int tid = threadIdx.x;
    const long long traj = blockIdx.y;
    const int n = a.n;
    const int kk = n < K ? n : K;           // digits inside the tile (host guarantees kk >= RBD)
    int nt_act = 1;
    for (int j = 0; j < kk - RBD; ++j) nt_act *= DIM;   // active threads = stride of the first register digit
    const int tsz = nt_act * R;
    c2* tile = reinterpret_cast<c2*>(smem_raw);
    double* tab = reinterpret_cast<double*>(smem_raw + (((size_t)tsz * 16 + 127) / 128) * 128);
    const int stride = gen_table_stride(n, a.n_drives);
    const long long base = (long long)blockIdx.x * tsz;
    const long long voff = traj * a.D;

    if (tid == 0) mbar_init(&mbar, 1);
    for (int i = tid; i < stride; i += blockDim.x) tab[i] = a.table[traj * stride + i];
    __syncthreads();
    if (tid == 0) {
        mbar_arrive_expect_tx(&mbar, (uint32_t)tsz * 16u);
        tma_load_1d(tile, a.v + voff + base, (uint32_t)tsz * 16u, &mbar);
    }
    if (tid < 32) {
        // partners across the digits above the tile: one lane per (digit, drive), compacted in order by ballot
        int cnt = 0;
        double dh = 0.0;
        const int total = (n - kk) * a.n_drives;
        for (int e0 = 0; e0 < total; e0 += 32) {
            const int e = e0 + tid;
            bool valid = false;
            TileExtra te = {0, 0.0, 0.0};
            if (e < total) {
                const int j = kk + e / a.n_drives, q = e % a.n_drives;
                long long rem = blockIdx.x, st = tsz;
                for (int jj = kk; jj < j; ++jj) { rem /= DIM; st *= DIM; }
                const int digit = (int)(rem % DIM);
                const int k = n - 1 - j;
                const double* gq = tab + q * 3 * n;
                if (digit == a.to[q]) {
                    valid = true;
                    te = {(long long)(a.from[q] - a.to[q]) * st, gq[2 * k], gq[2 * k + 1]};
                } else if (digit == a.from[q]) {
                    valid = true;
                    te = {(long long)(a.to[q] - a.from[q]) * st, gq[2 * k], -gq[2 * k + 1]};
                    dh -= gq[2 * n + k];
                }
            }
            const unsigned m = __ballot_sync(0xffffffffu, valid);
            if (valid) extra[cnt + __popc(m & ((1u << tid) - 1u))] = te;
            cnt += __popc(m);
        }
        for (int o = 16; o > 0; o >>= 1) dh += __shfl_xor_sync(0xffffffffu, dh, o);
        if (tid == 0) { n_extra = cnt; diag_high = dh; }
    }
    __syncthreads();
    mbar_wait(&mbar, 0);
    double dot0 = 0.0, dot1 = 0.0;
    const bool fuse = a.lz.vj != nullptr;
    LanczosCoef lc{0.0, 0.0, 0.0, 0.0};
    if (fuse) lc = lanczos_coef(a.lz, traj);
    if (tid < nt_act) {

    double rr[R], ri[R], dd[R];
#pragma unroll
    for (int i = 0; i < R; ++i) { rr[i] = 0.0; ri[i] = 0.0; dd[i] = 0.0; }
    double diag_low = 0.0;
    // --- the tile digits below the register block: selects once per (digit, drive), R shared-memory reads ---
    {
        int rem = tid, st = 1;
#pragma unroll
        for (int j = 0; j < K - RBD; ++j) {
            if (j < kk - RBD) {
                const int digit = rem % DIM;
                rem /= DIM;
                const int k = n - 1 - j;
                for (int q = 0; q < a.n_drives; ++q) {
                    const double* gq = tab + q * 3 * n;
                    const bool is_to = digit == a.to[q], is_from = digit == a.from[q];
                    if (is_to || is_from) {
                        const int off = tid + (is_to ? (a.from[q] - a.to[q]) : (a.to[q] - a.from[q])) * st;
                        const double gx = gq[2 * k];
                        const double gy = is_to ? gq[2 * k + 1] : -gq[2 * k + 1];
                        diag_low -= is_from ? gq[2 * n + k] : 0.0;
#pragma unroll
                        for (int i = 0; i < R; ++i) {
                            const c2 pv = tile[off + i * nt_act];
                            rr[i] = fma(gx, pv.x, rr[i]); rr[i] = fma(-gy, pv.y, rr[i]);
                            ri[i] = fma(gx, pv.y, ri[i]); ri[i] = fma(gy, pv.x, ri[i]);
                        }
                    }
                }
                st *= DIM;
            }
        }
    }
    // --- the register-block digits: the digit of amplitude i is a compile-time constant ---
#pragma unroll
    for (int jj = 0; jj < RBD; ++jj) {
        const int j = kk - RBD + jj;
        const int k = n - 1 - j;
        const int stj = nt_act * ipow_c(DIM, jj);
        for (int q = 0; q < a.n_drives; ++q) {
            const double* gq = tab + q * 3 * n;
            const double gx0 = gq[2 * k], gy0 = gq[2 * k + 1], th = gq[2 * n + k];
            const int to = a.to[q], from = a.from[q];
#pragma unroll
            for (int i = 0; i < R; ++i) {
                const int digit = (i / ipow_c(DIM, jj)) % DIM;
                const bool is_to = digit == to, is_from = digit == from;
                if (is_to || is_from) {   // uniform across the CTA
                    const c2 pv = tile[tid + i * nt_act + (is_to ? (from - to) : (to - from)) * stj];
                    const double gy = is_to ? gy0 : -gy0;
                    rr[i] = fma(gx0, pv.x, rr[i]); rr[i] = fma(-gy, pv.y, rr[i]);
                    ri[i] = fma(gx0, pv.y, ri[i]); ri[i] = fma(gy, pv.x, ri[i]);
                    dd[i] -= is_from ? th : 0.0;
                }
            }
        }
    }
    // --- the digits above the tile: CTA-uniform (offset, coefficient) list, coalesced loads ---
    const c2* vbase = a.v + voff + base + tid;
    const int nex = n_extra;
    for (int e = 0; e < nex; ++e) {
        const long long off = extra[e].off;
        const double gx = extra[e].gx, gy = extra[e].gy;
#pragma unroll
        for (int i = 0; i < R; ++i) {
            const double2 raw = __ldg(reinterpret_cast<const double2*>(vbase + off + i * nt_act));
            rr[i] = fma(gx, raw.x, rr[i]); rr[i] = fma(-gy, raw.y, rr[i]);
            ri[i] = fma(gx, raw.y, ri[i]); ri[i] = fma(gy, raw.x, ri[i]);
        }
    }
    // --- epilogue ---
    const double w = tab[stride - 2], gamma = tab[stride - 1];
    const c2 cb2 = a.beta_dev ? c2{-a.beta_dev[traj], 0.0} : a.coef.c_b2;
    const double dcommon = diag_high + diag_low - gamma;
    const double* dsrc = a.dint ? a.dint + traj * a.dint_stride : nullptr;
    constexpr int H = (R % 3 == 0) ? 3 : 4;
#pragma unroll
    for (int h0 = 0; h0 < R; h0 += H) {
        double dv[H];
        c2 pv[H], bv[H];
#pragma unroll
        for (int r = 0; r < H; ++r) {
            const long long idx = base + tid + (long long)(h0 + r) * nt_act;
            dv[r] = dsrc ? __ldcs(dsrc + idx) : 0.0;
            pv[r] = {0.0, 0.0}; bv[r] = {0.0, 0.0};
            if (fuse) {
                pv[r] = ld_own(a.lz.vj + voff + idx);
                if (a.lz.vjm1 && lc.beta_prev != 0.0) bv[r] = ld_own(a.lz.vjm1 + voff + idx);
            } else {
                if (a.psi) pv[r] = ld_own(a.psi + voff + idx);
                if (a.b2) bv[r] = ld_own(a.b2 + voff + idx);
            }
        }
#pragma unroll
        for (int r = 0; r < H; ++r) {
            const int i = h0 + r;
            const long long idx = base + tid + (long long)i * nt_act;
            const c2 vo = tile[tid + i * nt_act];
            const double diag = fma(w, dv[r], dcommon + dd[i]);
            const c2 gv = {fma(diag, vo.x, rr[i]), fma(diag, vo.y, ri[i])};
            c2 res, lhs;
            if (fuse) {   // fused Lanczos step (see LanczosFuse)
                const c2 vn = {(vo.x - lc.alpha * pv[r].x) * lc.inv, (vo.y - lc.alpha * pv[r].y) * lc.inv};
                const double ai = lc.alpha * lc.inv, abi = ai * lc.beta_prev;
                res.x = fma(lc.inv, gv.x, -fma(ai, vo.x, fma(abi, bv[r].x, lc.beta * pv[r].x)));
                res.y = fma(lc.inv, gv.y, -fma(ai, vo.y, fma(abi, bv[r].y, lc.beta * pv[r].y)));
                st_c2(a.lz.vout + voff + idx, vn);
                lhs = vn;
            } else {
                res = cmul(a.coef.c_g, gv);
                res = cadd(res, cmul(a.coef.c_psi, pv[r]));
                res = cadd(res, cmul(cb2, bv[r]));
                lhs = vo;
            }
            dot0 = fma(lhs.x, res.x, dot0); dot0 = fma(lhs.y, res.y, dot0);
            dot1 = fma(res.x, res.x, dot1); dot1 = fma(res.y, res.y, dot1);
            st_c2(a.out + voff + idx, res);
        }
    }
    }  // active threads
    if (a.dot_acc) {  // fused Lanczos inner products: warp __shfl reduction, one atomic pair per CTA
        for (int o = 16; o > 0; o >>= 1) {
            dot0 += __shfl_xor_sync(0xffffffffu, dot0, o);
            dot1 += __shfl_xor_sync(0xffffffffu, dot1, o);
        }
        __shared__ double dred[2][8];
        if ((tid & 31) == 0) { dred[0][tid >> 5] = dot0; dred[1][tid >> 5] = dot1; }
        __syncthreads();
        if (tid == 0) {
            double s0 = 0.0, s1 = 0.0;
#pragma unroll
            for (int i = 0; i < 8; ++i) { s0 += dred[0][i]; s1 += dred[1][i]; }
            atomicAdd(a.dot_acc + 2 * traj, s0);
            atomicAdd(a.dot_acc + 2 * traj + 1, s1);
        }
    }
    if (fuse && blockIdx.x == 0 && tid == 0) {
        a.lz.alpha_out[traj] = lc.alpha;
        a.lz.beta_out[traj] = lc.beta;
        a.lz.acc_clear[2 * traj] = 0.0;
        a.lz.acc_clear[2 * traj + 1] = 0.0;
    }
}

// ---- interaction diagonal ---------------------------------------------------
// Dint[s] = sum_{i<j} U_ij [digit_i == r][digit_j == r]
// (make_vdw_term, hamiltonian.py:260-274, after the + dag doubling of 0.5*U)
// Here and in the reductions below, `off` is the global index of element 0 (the first amplitude of a state-vector
// shard, 0 for a whole state): the digits are those of off + idx.
__global__ void dint_kernel(double* dint, const double* U, int n, int dim, int rstate, long long D, long long off) {
    extern __shared__ double Us[];
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) Us[i] = U[i];
    __syncthreads();
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < D;
         idx += (long long)gridDim.x * blockDim.x) {
        int pos[64];
        int cnt = 0;
        long long rem = off + idx;
        for (int k = n - 1; k >= 0; --k) {
            if ((int)(rem % dim) == rstate) pos[cnt++] = k;
            rem /= dim;
        }
        double acc = 0.0;
        // pos is descending in k; accumulate pairs in (i<j) order of the reference loop
        for (int a = cnt - 1; a >= 0; --a)
            for (int b = a - 1; b >= 0; --b) acc += Us[pos[a] * n + pos[b]];
        dint[idx] = acc;
    }
}

// min / max of Dint grouped by the number of |r> digits (spectral bounds)
__global__ void dint_bounds_kernel(const double* dint, int n, int dim, int rstate, long long D, double* mins,
                                   double* maxs, long long off) {
    // one thread per amplitude, atomics on (n+1) bins via ordered-int trick
    for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < D;
         idx += (long long)gridDim.x * blockDim.x) {
        int cnt = 0;
        long long rem = off + idx;
        for (int k = 0; k < n; ++k) { cnt += ((int)(rem % dim) == rstate); rem /= dim; }
        const double v = dint[idx];
        // Dint >= 0 is not guaranteed (negative C6 never occurs, but be safe): use CAS loops
        unsigned long long* pmin = reinterpret_cast<unsigned long long*>(mins + cnt);
        unsigned long long old = *pmin;
        while (__longlong_as_double((long long)old) > v) {
            unsigned long long assumed = old;
            old = atomicCAS(pmin, assumed, (unsigned long long)__double_as_longlong(v));
            if (old == assumed) break;
        }
        unsigned long long* pmax = reinterpret_cast<unsigned long long*>(maxs + cnt);
        old = *pmax;
        while (__longlong_as_double((long long)old) < v) {
            unsigned long long assumed = old;
            old = atomicCAS(pmax, assumed, (unsigned long long)__double_as_longlong(v));
            if (old == assumed) break;
        }
    }
}

// ---- measurement: bitstring weights, occupations, sampling ---------------------------------------------------
// The weight of basis state s in trajectory traj: |psi_s|^2 of a ket (RHO = false: D amplitudes per trajectory), or
// the diagonal element Re rho_ss of a density matrix (RHO = true: vec(rho)[r D + c] = rho_rc, D = the dimension of
// the physical register, `rows` rows of D entries per trajectory).  A density-matrix shard holds the rows
// [r0, r0 + rows) of one matrix: p = its slice + r0 points at rho[r0, r0], and s counts from r0.
template <bool RHO>
__device__ __forceinline__ double basis_weight(const c2* p, long long traj, long long D, long long rows, long long s) {
    if constexpr (RHO) {
        return p[traj * rows * D + s * (D + 1)].x;
    } else {
        const c2 v = p[traj * D + s];
        return v.x * v.x + v.y * v.y;
    }
}

// weights[b(s)] += |psi_s|^2 (or rho_ss) with bit k of b = [digit_k(s) == one_digit], qudit 0 = most significant bit
// (QutipResult._weights, qutip_result.py:101-158: reversal for ground-rydberg and the 3/4-level
// marginalisation are both this rule).  A shard (d = 2) covers an aligned block of 2^L = rows bitstrings:
// weights[b mod rows].  `rows` basis states from `off` on (rows = D but on a density-matrix shard, basis_weight).
// A density matrix's diagonal may carry rounding noise below zero: it is clipped so the cumulative sum stays monotone.
template <bool RHO>
__global__ void bitstring_weights_kernel(const c2* psi, double* weights, long long D, long long rows, int n, int dim,
                                         int one_digit, long long off) {
    for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < rows;
         s += (long long)gridDim.x * blockDim.x) {
        double p = basis_weight<RHO>(psi, 0, D, rows, s);
        if constexpr (RHO) p = fmax(p, 0.0);
        long long rem = off + s, b = 0;
        for (int k = n - 1; k >= 0; --k) {  // qudit k <-> bit n-1-k
            if ((int)(rem % dim) == one_digit) b |= 1LL << (n - 1 - k);
            rem /= dim;
        }
        if (dim == 2) weights[b & (rows - 1)] = p;  // a permutation: no atomics needed
        else atomicAdd(weights + b, p);
    }
}

// occ[k] += sum_s |psi_s|^2 [digit_k(s) == digit]   (Occupation observable / <n_k>; rho_ss for RHO; `rows` as in
// bitstring_weights_kernel)
template <bool RHO>
__global__ void occupation_kernel(const c2* psi, double* occ, long long D, long long rows, int n, int dim, int digit,
                                  long long off) {
    extern __shared__ double socc[];
    for (int i = threadIdx.x; i < n; i += blockDim.x) socc[i] = 0.0;
    __syncthreads();
    const long long traj = blockIdx.y;
    for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < rows;
         s += (long long)gridDim.x * blockDim.x) {
        const double p = basis_weight<RHO>(psi, traj, D, rows, s);
        if (p == 0.0) continue;
        long long rem = off + s;
        for (int k = n - 1; k >= 0; --k) {
            if ((int)(rem % dim) == digit) atomicAdd(&socc[k], p);
            rem /= dim;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) atomicAdd(occ + traj * n + i, socc[i]);
}

// corr[traj][i*n+j] (i <= j) += sum_s |psi_s|^2 [digit_i(s) == digit][digit_j(s) == digit]
// (CorrelationMatrix observable <n_i n_j>; the diagonal is the occupation).  A block stages 2048 probabilities and
// their per-qudit match masks in shared memory; each warp then reduces a subset of the n(n+1)/2 pairs over them.
// RHO: the weights are the diagonal rho_ss.  `rows` as in bitstring_weights_kernel.
template <bool RHO>
__global__ void __launch_bounds__(256) correlation_kernel(const c2* psi, double* corr, long long D, long long rows, int n,
                                                          int dim, int digit, long long off) {
    constexpr int CH = 2048;
    __shared__ double sp[CH];
    __shared__ unsigned long long sm[CH];
    const long long traj = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int npairs = n * (n + 1) / 2;
    for (long long base = blockIdx.x * (long long)CH; base < rows; base += (long long)gridDim.x * CH) {
        for (int e = threadIdx.x; e < CH; e += blockDim.x) {
            const long long s = base + e;
            double p = 0.0;
            unsigned long long m = 0ull;
            if (s < rows) {
                p = basis_weight<RHO>(psi, traj, D, rows, s);
                long long rem = off + s;
                for (int k = n - 1; k >= 0; --k) {
                    if ((int)(rem % dim) == digit) m |= 1ull << k;
                    rem /= dim;
                }
            }
            sp[e] = p; sm[e] = m;
        }
        __syncthreads();
        int i = 0, first = 0;  // pairs enumerated row by row: (0,0..n-1), (1,1..n-1), ...
        for (int pr = warp; pr < npairs; pr += nw) {
            while (pr - first >= n - i) { first += n - i; ++i; }
            const int j = i + (pr - first);
            const unsigned long long need = (1ull << i) | (1ull << j);
            double acc = 0.0;
            for (int e = lane; e < CH; e += 32)
                if ((sm[e] & need) == need) acc += sp[e];
            for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
            if (lane == 0 && acc != 0.0) atomicAdd(corr + traj * n * n + i * n + j, acc);
        }
        __syncthreads();
    }
}

// acc[traj] += <phi, psi_traj> (complex; phi shared by all trajectories)   (Fidelity observable / State.overlap)
__global__ void overlap_kernel(const c2* phi, const c2* psi, long long D, double* acc) {
    const long long traj = blockIdx.y;
    double re = 0.0, im = 0.0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x) {
        const c2 a = phi[i], b = psi[traj * D + i];
        re = fma(a.x, b.x, re); re = fma(a.y, b.y, re);
        im = fma(a.x, b.y, im); im = fma(-a.y, b.x, im);
    }
    for (int o = 16; o > 0; o >>= 1) {
        re += __shfl_xor_sync(0xffffffffu, re, o);
        im += __shfl_xor_sync(0xffffffffu, im, o);
    }
    __shared__ double ws[2][8];
    if ((threadIdx.x & 31) == 0) { ws[0][threadIdx.x >> 5] = re; ws[1][threadIdx.x >> 5] = im; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s0 = 0.0, s1 = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { s0 += ws[0][i]; s1 += ws[1][i]; }
        atomicAdd(acc + 2 * traj, s0);
        atomicAdd(acc + 2 * traj + 1, s1);
    }
}

// ---- expectation of an operator given as monomial terms (Expectation observable) --------------------------------
// A term is c (x)_{k in S} M_k with M_k[a, (a + m_k) mod d] = w_k[a]:
//     <psi|term|psi> = c sum_s conj(psi_s) prod_k w_k[s_k] psi_{s'},  s' = s with digit (s_k + m_k) mod d on S.
// The term table is staged through shared memory in chunks (chunk i: terms [chunk_t[i], chunk_t[i+1]) and site
// entries [chunk_s[i], chunk_s[i+1]), site offsets relative to the chunk), so any term count works.
constexpr int kExpChunkTerms = 256, kExpChunkSites = 256;

// d = 2: the host folds the site factors of a term into masks of the GLOBAL index g (shard offset + local index):
// partner g ^ f; zero unless (g & care) == val; sign (-1)^popc(g & z); times r_j for every general site j whose bit
// is set in g.  Terms arrive sorted by f, so one partner load serves every term of a run of equal masks.
struct ExpD2Term {
    c2 c;
    unsigned long long f, care, val, z;
    int s0, sn;  // general sites of the term in the staged chunk
};
struct ExpGenSite { c2 r; unsigned long long bit; };
// where the partners live: src[shard ^ (f >> local_bits)] holds the slice of index bits above local_bits (one
// pointer and shard 0 for a whole state; a shard group passes every shard's state, peers through peer access).
// row_len > 0: RHO on the rows a density-matrix shard holds (expect_terms_d2_kernel), rows of row_len entries
struct ExpSrc { const c2* p[8]; int shard; int local_bits; long long row_len; };

__device__ __forceinline__ void exp_reduce(double re, double im, double* acc) {
    for (int o = 16; o > 0; o >>= 1) {
        re += __shfl_xor_sync(0xffffffffu, re, o);
        im += __shfl_xor_sync(0xffffffffu, im, o);
    }
    __shared__ double ws[2][8];
    if ((threadIdx.x & 31) == 0) { ws[0][threadIdx.x >> 5] = re; ws[1][threadIdx.x >> 5] = im; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s0 = 0.0, s1 = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { s0 += ws[0][i]; s1 += ws[1][i]; }
        atomicAdd(acc + 2 * blockIdx.y, s0);
        atomicAdd(acc + 2 * blockIdx.y + 1, s1);
    }
}

// acc[traj] += sum_terms (blockIdx.y = trajectory; D = 2^local_bits amplitudes per trajectory; 256 threads).
// RHO: src.p[0] holds density matrices of D^2 entries (no shards) and the term reads Tr(term rho) =
// sum_g term[g, g ^ f] rho[g ^ f, g]: one element per (mask, g), never the whole matrix.  With src.row_len, the plan
// holds the D rows g = (shard << local_bits) | s of one matrix (a shard), and the same trace is summed over the stored
// rows instead: sum_g term[g ^ f, g] rho[g, g ^ f], the term's factors read at x = g ^ f.
template <bool RHO>
__global__ void __launch_bounds__(256) expect_terms_d2_kernel(const __grid_constant__ ExpSrc src, long long D,
                                                              const ExpD2Term* terms, const ExpGenSite* gens,
                                                              const int* chunk_t, const int* chunk_s, int n_chunks,
                                                              double* acc) {
    __shared__ ExpD2Term st[kExpChunkTerms];
    __shared__ ExpGenSite sg[kExpChunkSites];
    const long long traj_off = (long long)blockIdx.y * (RHO ? D * (src.row_len ? src.row_len : D) : D);
    const c2* own = src.p[src.shard] + traj_off;
    const unsigned long long off = (unsigned long long)src.shard << src.local_bits;
    const unsigned long long lmask = (unsigned long long)D - 1ull;
    double re = 0.0, im = 0.0;
    for (int ch = 0; ch < n_chunks; ++ch) {
        const int t0 = chunk_t[ch], nt = chunk_t[ch + 1] - t0, s0 = chunk_s[ch], ns = chunk_s[ch + 1] - s0;
        __syncthreads();  // the previous chunk is consumed
        for (int i = threadIdx.x; i < nt; i += blockDim.x) st[i] = terms[t0 + i];
        for (int i = threadIdx.x; i < ns; i += blockDim.x) sg[i] = gens[s0 + i];
        __syncthreads();
        for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < D; s += (long long)gridDim.x * blockDim.x) {
            const c2 v = RHO ? c2{0.0, 0.0} : own[s];
            const unsigned long long g = off | (unsigned long long)s;
            unsigned long long fcur = ~0ull;
            c2 q = {0.0, 0.0};  // conj(psi_g) psi_{g ^ f}, or rho[g ^ f, g]
            for (int t = 0; t < nt; ++t) {
                const ExpD2Term& T = st[t];
                if (T.f != fcur) {  // uniform across the block: the loads of a warp are coalesced
                    fcur = T.f;
                    if constexpr (RHO) {
                        q = src.row_len ? own[s * src.row_len + (long long)(g ^ fcur)]
                                        : own[(long long)((unsigned long long)s ^ fcur) * D + s];
                    } else {
                        c2 p = v;
                        if (fcur) p = src.p[src.shard ^ (int)(fcur >> src.local_bits)][traj_off + (long long)((unsigned long long)s ^ (fcur & lmask))];
                        q = {v.x * p.x + v.y * p.y, v.x * p.y - v.y * p.x};
                    }
                }
                const unsigned long long x = (RHO && src.row_len) ? g ^ fcur : g;   // the row of the term's element
                if ((x & T.care) != T.val) continue;
                c2 c = T.c;
                for (int j = 0; j < T.sn; ++j)
                    if (x & sg[T.s0 + j].bit) c = cmul(c, sg[T.s0 + j].r);
                if (__popcll(x & T.z) & 1) c = {-c.x, -c.y};
                re = fma(c.x, q.x, re); re = fma(-c.y, q.y, re);
                im = fma(c.x, q.y, im); im = fma(c.y, q.x, im);
            }
        }
    }
    exp_reduce(re, im, acc);
}

// d = 3 / 4: digit a = (s / stride) mod d of each site, factor w[a], partner digit (a + shift) mod d
struct ExpTerm { c2 c; int s0, sn; };
struct ExpSite { long long stride; int shift, pad; c2 w[4]; };

// RHO: psi holds density matrices of D^2 entries; the term with partner s' reads rho[s', s]
template <bool RHO>
__global__ void __launch_bounds__(256) expect_terms_kernel(const c2* psi, long long D, int dim, const ExpTerm* terms,
                                                           const ExpSite* sites, const int* chunk_t, const int* chunk_s,
                                                           int n_chunks, double* acc) {
    __shared__ ExpTerm st[kExpChunkTerms];
    __shared__ ExpSite ss[kExpChunkSites];
    const c2* v_traj = psi + (long long)blockIdx.y * (RHO ? D * D : D);
    double re = 0.0, im = 0.0;
    for (int ch = 0; ch < n_chunks; ++ch) {
        const int t0 = chunk_t[ch], nt = chunk_t[ch + 1] - t0, s0 = chunk_s[ch], ns = chunk_s[ch + 1] - s0;
        __syncthreads();
        for (int i = threadIdx.x; i < nt; i += blockDim.x) st[i] = terms[t0 + i];
        for (int i = threadIdx.x; i < ns; i += blockDim.x) ss[i] = sites[s0 + i];
        __syncthreads();
        for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < D; s += (long long)gridDim.x * blockDim.x) {
            const c2 v = RHO ? c2{0.0, 0.0} : v_traj[s];
            for (int t = 0; t < nt; ++t) {
                const ExpTerm& T = st[t];
                c2 c = T.c;
                long long sp = s;
                for (int j = 0; j < T.sn; ++j) {
                    const ExpSite& S = ss[T.s0 + j];
                    const int a = (int)((s / S.stride) % dim);
                    int b = a + S.shift;
                    if (b >= dim) b -= dim;
                    c = cmul(c, S.w[a]);
                    sp += (long long)(b - a) * S.stride;
                }
                if (c.x == 0.0 && c.y == 0.0) continue;
                c2 q;
                if constexpr (RHO) {
                    q = v_traj[sp * D + s];
                } else {
                    const c2 p = v_traj[sp];
                    q = {v.x * p.x + v.y * p.y, v.x * p.y - v.y * p.x};
                }
                re = fma(c.x, q.x, re); re = fma(-c.y, q.y, re);
                im = fma(c.x, q.y, im); im = fma(c.y, q.x, im);
            }
        }
    }
    exp_reduce(re, im, acc);
}

// ---- reductions of density matrices vec(rho)[r D + c] = rho[r, c] (D^2 entries per trajectory, blockIdx.y) -------
// A density-matrix shard holds the rows [r0, r0 + rows) of one matrix (rows = D, r0 = 0 for whole matrices): the sums
// below run over the rows a plan holds, so a shard's value is its share of the whole matrix's.
// acc[2 traj] += Re Tr rho  (rho: the slice + r0, basis_weight)
__global__ void __launch_bounds__(256) density_trace_kernel(const c2* rho, long long D, long long rows, double* acc) {
    double tr = 0.0;
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < rows; r += (long long)gridDim.x * blockDim.x)
        tr += basis_weight<true>(rho, blockIdx.y, D, rows, r);
    exp_reduce(tr, 0.0, acc);
}

// acc[traj] += <phi| rho |phi> = sum_{r,c} conj(phi_r) rho[r, c] phi_c (complex): a block per row at a time
__global__ void __launch_bounds__(256) density_overlap_kernel(const c2* phi, const c2* rho, long long D, long long rows,
                                                              long long r0, double* acc) {
    const c2* m = rho + (long long)blockIdx.y * rows * D;
    double re = 0.0, im = 0.0;
    for (long long r = blockIdx.x; r < rows; r += gridDim.x) {
        double sr = 0.0, si = 0.0;  // sum_c rho[r, c] phi_c
        for (long long c = threadIdx.x; c < D; c += blockDim.x) {
            const c2 a = m[r * D + c], b = phi[c];
            sr = fma(a.x, b.x, sr); sr = fma(-a.y, b.y, sr);
            si = fma(a.x, b.y, si); si = fma(a.y, b.x, si);
        }
        const c2 p = phi[r0 + r];  // conj(p) (sr + i si)
        re = fma(p.x, sr, re); re = fma(p.y, si, re);
        im = fma(p.x, si, im); im = fma(-p.y, sr, im);
    }
    exp_reduce(re, im, acc);
}

// H(t) of a single-state plan in the form the density reductions read it: per drive q and qudit k the element
// g[q][k] = H[.. to_q .., .. from_q ..] (conj(g) on the transposed pair) and the detuning th[q][k] entering as
// -th |from_q><from_q|_k; dint = the interaction diagonal (nullptr when there is none).  No XY exchange term.
constexpr int kDensityMaxQudits = 20;
struct DensityH {
    c2 g[PB200_MAX_DRIVES_K][kDensityMaxQudits];
    double th[PB200_MAX_DRIVES_K][kDensityMaxQudits];
    int to[PB200_MAX_DRIVES_K], from[PB200_MAX_DRIVES_K];
    int n, dim, n_drives;
    const double* dint;
};

// (H rho)[a, r] = sum_b H[a, b] rho[b, r] over the diagonal and the drive transitions of a; diag = H[a, a]
__device__ __forceinline__ c2 density_h_row(const DensityH& h, const c2* m, long long D, long long a, long long r,
                                            double& diag) {
    diag = h.dint ? h.dint[a] : 0.0;
    double yr = 0.0, yi = 0.0;
    long long rem = a, st = 1;
    for (int k = h.n - 1; k >= 0; --k) {  // qudit k has stride dim^(n-1-k)
        const int digit = (int)(rem % h.dim);
        rem /= h.dim;
        for (int q = 0; q < h.n_drives; ++q) {
            const c2 g = h.g[q][k];
            if (digit == h.to[q]) {
                const c2 v = m[(a + (long long)(h.from[q] - h.to[q]) * st) * D + r];
                yr = fma(g.x, v.x, yr); yr = fma(-g.y, v.y, yr);
                yi = fma(g.x, v.y, yi); yi = fma(g.y, v.x, yi);
            } else if (digit == h.from[q]) {
                const c2 v = m[(a + (long long)(h.to[q] - h.from[q]) * st) * D + r];
                yr = fma(g.x, v.x, yr); yr = fma(g.y, v.y, yr);
                yi = fma(g.x, v.y, yi); yi = fma(-g.y, v.x, yi);
                diag -= h.th[q][k];
            }
        }
        st *= h.dim;
    }
    const c2 v = m[a * D + r];
    return {fma(diag, v.x, yr), fma(diag, v.y, yi)};
}

// acc[2 traj] += Re Tr(H rho), acc[2 traj + 1] += Re Tr(H^2 rho):  per diagonal index r,
// (H rho)[r, r] and sum_a H[r, a] (H rho)[a, r] over a = r and the drive partners of r
__global__ void __launch_bounds__(256) density_energy_kernel(const c2* rho, long long D, const __grid_constant__ DensityH h,
                                                             double* acc) {
    const c2* m = rho + (long long)blockIdx.y * D * D;
    double e1 = 0.0, e2 = 0.0;
    for (long long r = blockIdx.x * (long long)blockDim.x + threadIdx.x; r < D; r += (long long)gridDim.x * blockDim.x) {
        double diag, unused;
        const c2 y = density_h_row(h, m, D, r, r, diag);
        e1 += y.x;
        e2 = fma(diag, y.x, e2);
        long long rem = r, st = 1;
        for (int k = h.n - 1; k >= 0; --k) {
            const int digit = (int)(rem % h.dim);
            rem /= h.dim;
            for (int q = 0; q < h.n_drives; ++q) {
                c2 g = h.g[q][k];  // H[r, a]
                long long a;
                if (digit == h.to[q]) a = r + (long long)(h.from[q] - h.to[q]) * st;
                else if (digit == h.from[q]) { a = r + (long long)(h.to[q] - h.from[q]) * st; g.y = -g.y; }
                else continue;
                const c2 ya = density_h_row(h, m, D, a, r, unused);
                e2 = fma(g.x, ya.x, e2); e2 = fma(-g.y, ya.y, e2);
            }
            st *= h.dim;
        }
    }
    exp_reduce(e1, e2, acc);
}

// (rho H)[b, a] = sum_c rho[b, c] H[c, a] over c = a and the drive transitions of a, from row b of rho alone (m + b D:
// the row as the plan stores it); diag = H[a, a].  H[c, a] = conj(H[a, c]): the elements density_h_row reads, conjugated
__device__ __forceinline__ c2 density_row_h(const DensityH& h, const c2* row, long long a, double& diag) {
    diag = h.dint ? h.dint[a] : 0.0;
    double yr = 0.0, yi = 0.0;
    long long rem = a, st = 1;
    for (int k = h.n - 1; k >= 0; --k) {
        const int digit = (int)(rem % h.dim);
        rem /= h.dim;
        for (int q = 0; q < h.n_drives; ++q) {
            const c2 g = h.g[q][k];
            if (digit == h.to[q]) {   // H[c, a] = H[.. from .., .. to ..] = conj(g)
                const c2 v = row[a + (long long)(h.from[q] - h.to[q]) * st];
                yr = fma(g.x, v.x, yr); yr = fma(g.y, v.y, yr);
                yi = fma(g.x, v.y, yi); yi = fma(-g.y, v.x, yi);
            } else if (digit == h.from[q]) {   // H[c, a] = g
                const c2 v = row[a + (long long)(h.to[q] - h.from[q]) * st];
                yr = fma(g.x, v.x, yr); yr = fma(-g.y, v.y, yr);
                yi = fma(g.x, v.y, yi); yi = fma(g.y, v.x, yi);
                diag -= h.th[q][k];
            }
        }
        st *= h.dim;
    }
    const c2 v = row[a];
    return {fma(diag, v.x, yr), fma(diag, v.y, yi)};
}

// The rows [r0, r0 + rows) of one density matrix (a shard's): acc[0] += Re sum_b (rho H)[b, b], acc[1] += Re sum_b
// sum_a (rho H)[b, a] H[a, b] over a = b and the drive partners of b.  Tr(H rho) = Tr(rho H) and Tr(H^2 rho) =
// Tr(rho H^2): the same sums as density_energy_kernel's, ordered so that every element read lies in a stored row.
__global__ void __launch_bounds__(256) density_energy_rows_kernel(const c2* rho, long long D, long long rows, long long r0,
                                                                  const __grid_constant__ DensityH h, double* acc) {
    double e1 = 0.0, e2 = 0.0;
    for (long long bl = blockIdx.x * (long long)blockDim.x + threadIdx.x; bl < rows; bl += (long long)gridDim.x * blockDim.x) {
        const long long b = r0 + bl;
        const c2* row = rho + bl * D;
        double diag, unused;
        const c2 y = density_row_h(h, row, b, diag);
        e1 += y.x;
        e2 = fma(diag, y.x, e2);
        long long rem = b, st = 1;
        for (int k = h.n - 1; k >= 0; --k) {
            const int digit = (int)(rem % h.dim);
            rem /= h.dim;
            for (int q = 0; q < h.n_drives; ++q) {
                c2 g = h.g[q][k];  // H[a, b]
                long long a;
                if (digit == h.to[q]) { a = b + (long long)(h.from[q] - h.to[q]) * st; g.y = -g.y; }
                else if (digit == h.from[q]) a = b + (long long)(h.to[q] - h.from[q]) * st;
                else continue;
                const c2 ya = density_row_h(h, row, a, unused);
                e2 = fma(g.x, ya.x, e2); e2 = fma(-g.y, ya.y, e2);
            }
            st *= h.dim;
        }
    }
    exp_reduce(e1, e2, acc);
}

// indices[i] = first j with cum[j] >= u[i] * total  (np.searchsorted(cumsum(w / sum w), rnd), side="left")
__global__ void search_sorted_kernel(const double* cum, long long M, const double* u, long long* idx, int n_shots) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_shots) return;
    const double target = u[i] * cum[M - 1];
    long long lo = 0, hi = M;  // first index with cum >= target
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (cum[mid] < target) lo = mid + 1; else hi = mid;
    }
    idx[i] = lo < M ? lo : M - 1;
}

// ---- small utilities --------------------------------------------------------
__global__ void set_basis_kernel(c2* psi, long long D, long long index) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x)
        psi[i] = {i == index ? 1.0 : 0.0, 0.0};
}

__global__ void prob_kernel(const c2* psi, double* probs, long long total) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const c2 v = psi[i];
        probs[i] = v.x * v.x + v.y * v.y;
    }
}

// squared norm per trajectory: grid.y = trajectory, warp-shuffle + one atomic per block
__global__ void norm2_kernel(const c2* psi, long long D, double* out) {
    const long long traj = blockIdx.y;
    double acc = 0.0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x) {
        const c2 v = psi[traj * D + i];
        acc = fma(v.x, v.x, acc);
        acc = fma(v.y, v.y, acc);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ double ws[8];
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += ws[i];
        atomicAdd(out + traj, s);
    }
}

// ---- dissipator of the Lindblad equation on the vectorised density matrix ------------------------------
// rho is stored as the state of 2N qudits (row digits above column digits).  A single-qudit collapse
// operator couples only the (row digit, column digit) pair of its qudit, so exp(h*D) factorises into one
// d^2 x d^2 matrix per qudit, applied in place to the pair of digits at strides s_hi > s_lo.
struct PairOp {
    c2 m[81];  // row-major [d*d][d*d], d <= 3
};

__global__ void pair_op_kernel(c2* psi, long long D, int dim, long long s_hi, long long s_lo,
                               const __grid_constant__ PairOp op) {
    const int dd = dim * dim;
    const long long groups = D / dd;
    const long long traj = blockIdx.y;
    c2* base = psi + traj * D;
    const long long mid_span = s_hi / (s_lo * dim);
    for (long long gidx = blockIdx.x * (long long)blockDim.x + threadIdx.x; gidx < groups;
         gidx += (long long)gridDim.x * blockDim.x) {
        long long q = gidx;
        const long long low = q % s_lo; q /= s_lo;
        const long long mid = q % mid_span; q /= mid_span;
        const long long idx0 = low + mid * s_lo * dim + q * s_hi * dim;
        c2 v[9], w[9];
        for (int a = 0; a < dim; ++a)
            for (int b = 0; b < dim; ++b) v[a * dim + b] = base[idx0 + a * s_hi + b * s_lo];
        for (int r = 0; r < dd; ++r) {
            double xr = 0.0, xi = 0.0;
            for (int c = 0; c < dd; ++c) {
                const c2 mm = op.m[r * dd + c];
                xr = fma(mm.x, v[c].x, xr); xr = fma(-mm.y, v[c].y, xr);
                xi = fma(mm.x, v[c].y, xi); xi = fma(mm.y, v[c].x, xi);
            }
            w[r] = {xr, xi};
        }
        for (int a = 0; a < dim; ++a)
            for (int b = 0; b < dim; ++b) base[idx0 + a * s_hi + b * s_lo] = w[a * dim + b];
    }
}

// ---- Lanczos (Krylov) propagator helpers ------------------------------------------------------------------
// acc[traj][0] += Re<v, w>, acc[traj][1] += <w, w>   (warp __shfl reduction, one atomic pair per block)
__global__ void dot2_kernel(const c2* v, const c2* w, long long D, double* acc) {
    const long long traj = blockIdx.y;
    double a0 = 0.0, a1 = 0.0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x) {
        const c2 x = v[traj * D + i], y = w[traj * D + i];
        a0 = fma(x.x, y.x, a0); a0 = fma(x.y, y.y, a0);
        a1 = fma(y.x, y.x, a1); a1 = fma(y.y, y.y, a1);
    }
    for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    __shared__ double ws[2][8];
    if ((threadIdx.x & 31) == 0) { ws[0][threadIdx.x >> 5] = a0; ws[1][threadIdx.x >> 5] = a1; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double s0 = 0.0, s1 = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { s0 += ws[0][i]; s1 += ws[1][i]; }
        atomicAdd(acc + 2 * traj, s0);
        atomicAdd(acc + 2 * traj + 1, s1);
    }
}

// w <- (w - alpha v) / beta with alpha = acc[0], beta = sqrt(acc[1] - alpha^2); records alpha, beta
// (beta = 0 and w = 0 on breakdown) and clears the accumulator of the other parity for the next iteration.
__global__ void lanczos_update_kernel(c2* w, const c2* v, long long D, const double* acc, double* alpha_out,
                                      double* beta_out, double* acc_clear) {
    const long long traj = blockIdx.y;
    const double alpha = acc[2 * traj];
    const double ww = acc[2 * traj + 1];
    const double b2 = ww - alpha * alpha;
    const double beta = (b2 > 1e-28 * fmax(ww, 1e-300)) ? sqrt(b2) : 0.0;
    const double inv = beta > 0.0 ? 1.0 / beta : 0.0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x) {
        const c2 x = v[traj * D + i];
        c2 y = w[traj * D + i];
        y.x = (y.x - alpha * x.x) * inv;
        y.y = (y.y - alpha * x.y) * inv;
        w[traj * D + i] = y;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        alpha_out[traj] = alpha;
        beta_out[traj] = beta;
        acc_clear[2 * traj] = 0.0;
        acc_clear[2 * traj + 1] = 0.0;
    }
}

// v0 <- psi / ||psi|| with ||psi||^2 = acc[1]; records the norm
__global__ void normalize_copy_kernel(c2* v0, const c2* psi, long long D, const double* acc, double* norm_out,
                                      double* acc_clear) {
    const long long traj = blockIdx.y;
    const double nrm = sqrt(acc[2 * traj + 1]);
    const double inv = nrm > 0.0 ? 1.0 / nrm : 0.0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x) {
        const c2 x = psi[traj * D + i];
        v0[traj * D + i] = {x.x * inv, x.y * inv};
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        norm_out[traj] = nrm;
        acc_clear[2 * traj] = 0.0;
        acc_clear[2 * traj + 1] = 0.0;
    }
}

// out = sum_j y[traj][j] V_j   (V_j = V + j * vstride; y interleaved complex [traj][m])
__global__ void krylov_combine_kernel(c2* out, const c2* V, long long vstride, long long D, const double* y, int m) {
    const long long traj = blockIdx.y;
    const double* yt = y + 2 * (long long)m * traj;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x) {
        double xr = 0.0, xi = 0.0;
        for (int j = 0; j < m; ++j) {
            const c2 v = V[j * vstride + traj * D + i];
            const double yr = yt[2 * j], yi = yt[2 * j + 1];
            xr = fma(yr, v.x, xr); xr = fma(-yi, v.y, xr);
            xi = fma(yr, v.y, xi); xi = fma(yi, v.x, xi);
        }
        out[traj * D + i] = {xr, xi};
    }
}

// ---- Monte-Carlo wave function: non-Hermitian decay and quantum jumps ---------------------------------------------
// psi[s] *= exp(-h/2 * sum_k gamma[digit_k(s)])  -- the diagonal part -i/2 sum L^+L of H_eff
struct DecayTable { double gamma[4]; };
__global__ void mcwf_decay_kernel(c2* psi, long long D, int n, int dim, double half_h, const __grid_constant__ DecayTable tb) {
    const long long traj = blockIdx.y;
    for (long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x; s < D;
         s += (long long)gridDim.x * blockDim.x) {
        long long rem = s;
        double acc = 0.0;
        for (int k = 0; k < n; ++k) { acc += tb.gamma[(int)(rem % dim)]; rem /= dim; }
        const double f = exp(-half_h * acc);
        c2 v = psi[traj * D + s];
        v.x *= f; v.y *= f;
        psi[traj * D + s] = v;
    }
}

// psi <- scale * (L on qudit with stride `st`) psi for one trajectory; L row-major d x d
struct QuditOp { c2 m[16]; };
__global__ void qudit_op_kernel(c2* psi, long long D, int dim, long long st, double scale, const __grid_constant__ QuditOp op) {
    psi += (long long)blockIdx.y * D;   // gridDim.y = trajectories (1 for a single-trajectory jump)
    const long long groups = D / dim;
    for (long long gidx = blockIdx.x * (long long)blockDim.x + threadIdx.x; gidx < groups;
         gidx += (long long)gridDim.x * blockDim.x) {
        const long long low = gidx % st, high = gidx / st;
        const long long idx0 = low + high * st * dim;
        c2 v[4], w[4];
        for (int a = 0; a < dim; ++a) v[a] = psi[idx0 + a * st];
        for (int r = 0; r < dim; ++r) {
            double xr = 0.0, xi = 0.0;
            for (int c = 0; c < dim; ++c) {
                const c2 mm = op.m[r * dim + c];
                xr = fma(mm.x, v[c].x, xr); xr = fma(-mm.y, v[c].y, xr);
                xi = fma(mm.x, v[c].y, xi); xi = fma(mm.y, v[c].x, xi);
            }
            w[r] = {xr * scale, xi * scale};
        }
        for (int a = 0; a < dim; ++a) psi[idx0 + a * st] = w[a];
    }
}

// Single-qudit reduced density matrix rho[a][b] = sum_rest psi(a, rest) conj(psi(b, rest)) of the qudit with stride
// `st` (one trajectory), accumulated into acc[2 * (a * dim + b) + {0, 1}]: the jump weights <L^+L> of a general
// (non-diagonal L^+L) collapse operator are Tr(L^+L rho) (hamiltonian.py:97-124 builds the operators).
__global__ void reduced_density_kernel(const c2* psi, long long D, int dim, long long st, double* acc) {
    const long long groups = D / dim;
    double re[16], im[16];
    for (int i = 0; i < 16; ++i) { re[i] = 0.0; im[i] = 0.0; }
    for (long long gidx = blockIdx.x * (long long)blockDim.x + threadIdx.x; gidx < groups;
         gidx += (long long)gridDim.x * blockDim.x) {
        const long long low = gidx % st, high = gidx / st;
        const long long idx0 = low + high * st * dim;
        c2 v[4];
        for (int a = 0; a < dim; ++a) v[a] = psi[idx0 + a * st];
        for (int a = 0; a < dim; ++a)
            for (int b = 0; b < dim; ++b) {
                re[a * dim + b] = fma(v[a].x, v[b].x, fma(v[a].y, v[b].y, re[a * dim + b]));
                im[a * dim + b] = fma(v[a].y, v[b].x, fma(-v[a].x, v[b].y, im[a * dim + b]));
            }
    }
    for (int i = 0; i < dim * dim; ++i) {
        double x = re[i], y = im[i];
        for (int o = 16; o > 0; o >>= 1) {
            x += __shfl_xor_sync(0xffffffffu, x, o);
            y += __shfl_xor_sync(0xffffffffu, y, o);
        }
        if ((threadIdx.x & 31) == 0) { atomicAdd(acc + 2 * i, x); atomicAdd(acc + 2 * i + 1, y); }
    }
}

__global__ void scale_kernel(c2* psi, long long D, double scale) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x) {
        c2 v = psi[i];
        psi[i] = {v.x * scale, v.y * scale};
    }
}

// y = alpha*y + beta*x (Richardson combination of the step-doubling pair)
__global__ void axpby_kernel(c2* y, const c2* x, double alpha, double beta, long long total) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const c2 a = y[i], b = x[i];
        y[i] = {alpha * a.x + beta * b.x, alpha * a.y + beta * b.y};
    }
}

// squared distance per trajectory (step-doubling error estimate)
__global__ void diffnorm2_kernel(const c2* a, const c2* b, long long D, double* out) {
    const long long traj = blockIdx.y;
    double acc = 0.0;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < D;
         i += (long long)gridDim.x * blockDim.x) {
        const c2 x = a[traj * D + i], y = b[traj * D + i];
        const double dr = x.x - y.x, di = x.y - y.y;
        acc = fma(dr, dr, acc);
        acc = fma(di, di, acc);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    __shared__ double ws[8];
    if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += ws[i];
        atomicAdd(out + traj, s);
    }
}

}  // namespace pb200
