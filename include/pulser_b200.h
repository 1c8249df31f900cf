/*
 * pulser_b200 -- C ABI of the H100-native (sm_90a) time-evolution hot path.
 *
 * The reference (pasqal-io/Pulser) is pure Python and has no FFI: its "plugin
 * boundary" for this path is the pair
 *     Hamiltonian(samples, noise_trajectory, basis_data, lindblad_data, rate)
 *         pulser-simulation/pulser_simulation/hamiltonian.py:45-81
 *     QutipEmulator._run_solver(hamiltonian, ...) -> qutip.sesolve/mesolve/mcsolve
 *         pulser-simulation/pulser_simulation/simulation.py:689-766
 * Every entry point below names the reference interface it replaces.
 *
 * Conventions
 *   - plain C types only; complex numbers are interleaved (re, im) doubles;
 *   - all pointers are HOST pointers owned by the caller unless the name says
 *     "device"; the library owns every device buffer inside the opaque plan;
 *   - every function returns PB200_OK (0) or a negative error code and never
 *     throws across the boundary; pb200_last_error() gives the message of the
 *     last failure on the calling thread;
 *   - a plan is bound to one CUDA device and one stream; a plan is not
 *     thread-safe, distinct plans are independent;
 *   - state index: qudit 0 is the most significant digit (big-endian), digit
 *     value = position in `eigenbasis` order (u,d,r,g,h,x subset), exactly as
 *     qutip.tensor builds it at hamiltonian.py:169-200.
 */
#ifndef PULSER_B200_H
#define PULSER_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PB200_OK 0
#define PB200_ERR_INVALID -1   /* bad argument */
#define PB200_ERR_CUDA -2      /* CUDA runtime failure (no device, OOM, ...) */
#define PB200_ERR_UNSUPPORTED -3
#define PB200_ERR_STATE -4     /* call order */

#define PB200_MAX_QUDITS 40
#define PB200_MAX_DRIVES 3

typedef struct pb200_plan pb200_plan; /* opaque */

/* One addressed basis: drive operator c(t)|to><from| + h.c. and detuning
 * -det(t)|from><from| on every qudit (hamiltonian.py:340-352, 370-375):
 * ground-rydberg: to=g, from=r; digital: to=h, from=g; XY: to=u, from=d. */
typedef struct pb200_drive_desc {
    int32_t state_to;    /* digit value of the |to> eigenstate   */
    int32_t state_from;  /* digit value of the |from> eigenstate */
    int32_t uniform;     /* 1: one table row shared by all qudits (Global) */
    int32_t reserved;
} pb200_drive_desc;

/* Static description: replaces the arguments of Hamiltonian.__init__
 * (hamiltonian.py:45-81) that do not change between noise trajectories. */
typedef struct pb200_plan_desc {
    int32_t n_qudits;       /* N */
    int32_t dim;            /* d = len(eigenbasis): 2, 3 or 4 */
    int32_t n_times;        /* len(sampling_times) */
    int32_t interp_order;   /* QobjEvo array-coefficient interpolation: 0 step,
                               1 linear, 3 cubic not-a-knot spline (QuTiP 5
                               default; hamiltonian.py:436) */
    int32_t n_drives;       /* addressed bases, <= PB200_MAX_DRIVES */
    int32_t rydberg_state;  /* digit of |r> for the U_ij n_i n_j term
                               (hamiltonian.py:260-274); -1: no interaction */
    int32_t n_traj;         /* trajectories evolved together (batch B >= 1) */
    int32_t device;         /* CUDA device ordinal */
    const double* sampling_times; /* [n_times] microseconds, increasing */
    pb200_drive_desc drives[PB200_MAX_DRIVES];
} pb200_plan_desc;

/* Integrator options (replace the `**options` handed to QuTiP at
 * simulation.py:800-845: max_step / nsteps / atol / rtol have no meaning for
 * the fixed-order propagator and are accepted-and-ignored on the Python side). */
typedef struct pb200_run_opts {
    int32_t max_step_samples; /* K: longest Magnus step, in sampling intervals
                                 (>=1). 0 = library default (32 adaptive+extrapolated,
                                 16 adaptive, 4 fixed). */
    int32_t refine_window;    /* steps are 1 interval long within this many
                                 intervals of a non-smooth sample; <0 = default */
    double cheb_tol;          /* Chebyshev truncation tolerance per exponential;
                                 0 = default (1e-12) */
    double rough_tol;         /* relative 3rd-difference threshold that marks a
                                 sample as non-smooth; 0 = default */
    int32_t magnus_order;     /* 2 or 4 (default 4) */
    int32_t check_every;      /* adaptive mode: smooth steps between two
                                 step-doubling checks; 0 = default (12) */
    double tol;               /* > 0: adaptive Magnus step, target 2-norm error of
                                 the state accumulated over the whole sampling-
                                 time range; 0 = default (1e-8); < 0: fixed steps
                                 of max_step_samples intervals */
    int32_t extrapolate;      /* 0 / 1 (default): every smooth step is a step-doubling
                                 pair combined by Richardson extrapolation (6th
                                 order); -1: plain 4th-order steps */
    int32_t integrator;       /* 1 Chebyshev-Clenshaw / 2 Lanczos (Krylov) exponentials of
                                 Richardson-CF4 Magnus steps; 3 time-dependent Taylor
                                 series (one global drive, its phase constant or
                                 moving, d = 2, one state: no Magnus error, ~1
                                 H-apply per ns on C2; also the master equation
                                 of a dissipator plan whose atoms share one
                                 generator without single-bit flips -- dephasing,
                                 relaxation, depolarizing -- under a drive of
                                 constant phase, with the dissipator inside the
                                 series and a default tol of 1e-10 instead of
                                 the splitting path's 1e-6; anything else with
                                 integrator 3 is PB200_ERR_UNSUPPORTED, reason
                                 given);
                                 0 auto: 3 where it applies, else 2 for strongly
                                 blockaded / HBM-resident registers, else 1.
                                 1 / 2 on a dissipator plan: Strang splitting of
                                 the dissipator around the Magnus steps */
} pb200_run_opts;

typedef struct pb200_run_stats {
    int64_t n_steps;        /* Magnus steps taken */
    int64_t n_exponentials; /* matrix exponentials applied */
    int64_t n_applies;      /* H-applies (Chebyshev terms), per trajectory */
    int64_t n_launches;     /* CUDA kernel launches */
    double gpu_ms;          /* device time of the propagation (CUDA events) */
    double max_rho;         /* largest Chebyshev half-width encountered */
    int64_t n_checks;       /* step-doubling checks performed (adaptive mode) */
    double err_estimate;    /* accumulated local-error estimate (adaptive mode) */
    double mean_step_samples; /* average smooth-step length, in sampling intervals */
    int64_t integrator;     /* 1 Chebyshev, 2 Lanczos, 3 Taylor: what the run used */
    int64_t n_rejected;     /* checked steps redone with a shorter step (adaptive mode) */
} pb200_run_stats;

int pb200_version(void);
const char* pb200_last_error(void);
/* number of visible CUDA devices (0 when there is none; never fails) */
int pb200_device_count(void);

/* ---- plan life cycle ---------------------------------------------------- */
int pb200_plan_create(pb200_plan** out, const pb200_plan_desc* desc);
int pb200_plan_destroy(pb200_plan* plan);
/* Use an existing CUDA stream (cudaStream_t passed as void*); NULL = the
 * plan's own stream. */
int pb200_plan_set_stream(pb200_plan* plan, void* cuda_stream);

/* Interaction matrix of trajectories [traj0, traj0+count): U[count][N][N]
 * (rad/us; only the strict upper triangle is read) and bad-atom mask
 * bad[count][N] (may be NULL = all good).  Replaces
 * noise_trajectory.interaction_matrix / bad_atoms as consumed by
 * make_vdw_term / make_interaction_term (hamiltonian.py:260-331).
 * shared != 0: the same matrix for every trajectory (count must be 1). */
int pb200_plan_set_interaction(pb200_plan* plan, int32_t traj0, int32_t count,
                               const double* U, const uint8_t* bad,
                               int32_t shared);

/* XY mode (microwave channel, eigenbasis u, d): exchange couplings
 * Uxy[count][N][N] of  Uxy_ij (|u d><d u| + h.c.)  (make_xy_term,
 * hamiltonian.py:276-294; interaction_matrix[0] in XY mode).  The |uu><uu| term
 * of the same function goes through pb200_plan_set_interaction with
 * rydberg_state = digit of |u>.  The SLM-mask time dependence (:399-424) is set with
 * pb200_plan_set_slm_mask.  shared != 0: one matrix for all trajectories. */
int pb200_plan_set_xy(pb200_plan* plan, int32_t traj0, int32_t count,
                      const double* Uxy, const uint8_t* bad, int32_t shared,
                      int32_t digit_u, int32_t digit_d);

/* XY mode with an SLM mask (hamiltonian.py:399-424): the interaction of every pair that contains a masked
 * qudit (masked[N] != 0) is multiplied by the interpolated coefficient coeff[n_times] -- the 0/1 array the
 * reference builds at :405-407 (0 up to the end of the mask, 1 afterwards) after _adapt_to_sampling_rate --
 * while the other pairs keep weight 1; i.e. H_int(t) = c(t) H_all + (1 - c(t)) H_unmasked, both terms spline-
 * interpolated like every QobjEvo coefficient.  Must be called before pb200_plan_set_interaction /
 * pb200_plan_set_xy (which split their matrices accordingly); one mask for all trajectories. */
int pb200_plan_set_slm_mask(pb200_plan* plan, const uint8_t* masked, const double* coeff);

/* Sample tables of drive `drive` for trajectories [traj0, traj0+count):
 *   coef[count][rows][n_times][2]  = 0.5*amp*exp(-i*phase)   (re, im)
 *   det [count][rows][n_times]     = detuning (enters H as -det |from><from|)
 * rows = 1 if the drive is uniform else N.  Replaces build_coeffs_ops
 * (hamiltonian.py:333-389). */
int pb200_plan_set_drive(pb200_plan* plan, int32_t drive, int32_t traj0,
                         int32_t count, const double* coef, const double* det);

/* Lindblad master equation (replaces qutip.mesolve(H, rho0, tlist, c_ops),
 * simulation.py:724-735).  The plan must describe the VECTORISED density matrix
 * as a system of 2N qudits: qudits 0..N-1 = row digits evolving under H,
 * qudits N..2N-1 = column digits evolving under -H^T (drive -conj(c), detuning
 * -det, interaction -U); the Python layer builds that description
 * (pulser_b200/lindblad.py).  `generators` holds, for each of the n_pairs = N
 * qudits, the d^2 x d^2 superoperator  sum_L ( L (x) conj(L) - 1/2 L^+L (x) 1
 * - 1/2 1 (x) (L^+L)^T )  of its collapse operators (hamiltonian.py:97-124),
 * row-major, interleaved complex, acting on the (row digit, column digit) pair
 * (k, k + N).  Afterwards pb200_propagate integrates  rho' = -i[H,rho] + D(rho)
 * by symmetric splitting  exp(h/2 D) U(h) exp(h/2 D)  with Richardson
 * extrapolation and the same step controller (order 2 -> 4).  d <= 3.
 * On a shard of vec(rho) (pb200_plan_create_shard of the 2N-qudit description:
 * the shard bits are the top row bits) every shard takes the same generators
 * before pb200_shards_link; pb200_shards_propagate then runs the Taylor
 * propagator with the dissipator inside the series. */
int pb200_plan_set_dissipator(pb200_plan* plan, int32_t n_pairs,
                              const double* generators);

/* Monte-Carlo wave function (replaces qutip.mcsolve(H, psi0, tlist, c_ops, ntraj),
 * simulation.py:710-735) for registers whose density matrix does not fit:
 * `ops` = n_ops single-qudit collapse matrices (d x d, row-major, interleaved
 * complex, coefficient included), each acting on every qudit
 * (hamiltonian.py:97-124).  When every L^+L is diagonal (dephasing, relaxation,
 * depolarizing, transition/projector-type effective noise) the no-jump decay is one
 * elementwise kernel and the jump weights come from the per-qudit populations; general
 * operators use exp(-tau sum L^+L) applied qudit by qudit and the single-qudit reduced
 * density matrices.  Afterwards
 * pb200_propagate evolves every trajectory under
 * H_eff = H - i/2 sum L^+L (symmetric splitting around the unitary step), and
 * applies a quantum jump whenever a trajectory's squared norm falls below its
 * random threshold (jump channel drawn from the <L^+L> weights; time resolution
 * = one step); states are renormalised at the end of the call. */
int pb200_plan_set_collapse(pb200_plan* plan, int32_t n_ops, const double* ops,
                            uint64_t seed);
/* number of quantum jumps applied so far, jumps[n_traj] */
int pb200_plan_jump_counts(pb200_plan* plan, int64_t* jumps);

/* ---- state --------------------------------------------------------------- */
/* Upload initial states psi[count][D] (interleaved complex); psi == NULL sets
 * basis state `basis_index` (e.g. all-ground, simulation.py:498-505) for the
 * given trajectories.  `broadcast` != 0: psi holds ONE state copied to all. */
int pb200_state_set(pb200_plan* plan, int32_t traj0, int32_t count,
                    const double* psi, int64_t basis_index, int32_t broadcast);
/* Download current states into psi[count][D]. */
int pb200_state_get(pb200_plan* plan, int32_t traj0, int32_t count, double* psi);
/* |psi|^2 summed into probs[count][D] (one array per trajectory). */
int pb200_state_probabilities(pb200_plan* plan, int32_t traj0, int32_t count,
                              double* probs);
/* squared norms, norms2[count] */
int pb200_state_norm2(pb200_plan* plan, int32_t traj0, int32_t count,
                      double* norms2);
/* Populations: occ[count][N], occ[t][k] = sum_s |psi_s|^2 [digit_k(s) == digit]
 * (the Occupation observable; default_observables.py:377-436). */
int pb200_state_occupation(pb200_plan* plan, int32_t traj0, int32_t count,
                           int32_t digit, double* occ);
/* <n_i n_j> of the current states, n_k = |digit><digit| on qudit k:
 * corr[count][N][N] (symmetric; the diagonal is the occupation).  Replaces the
 * CorrelationMatrix / Occupation observables' per-pair operator products
 * (pulser-core/pulser/backend/default_observables.py:331-428). */
int pb200_state_correlation(pb200_plan* plan, int32_t traj0, int32_t count,
                            int32_t digit, double* corr);

/* energy[b] = <psi_b|H_b(t)|psi_b>, h2[b] = <psi_b|H_b(t)^2|psi_b> for every
 * trajectory of the plan (Energy, EnergyVariance, EnergySecondMoment:
 * default_observables.py:431-561). */
int pb200_state_energy(pb200_plan* plan, double t_us, double* energy, double* h2);

/* out[c] = <phi|psi_{traj0+c}> as (re, im); phi: complex128[D] on the host
 * (Fidelity observable / State.overlap, default_observables.py:184-243). */
int pb200_state_overlap(pb200_plan* plan, int32_t traj0, int32_t count,
                        const double* phi, double* out);

/* An operator as a sum of monomial terms (Expectation observable,
 * default_observables.py:240-288, on an operator of Pulser's operator
 * representation, qutip_op.py:148-218).  Term t is
 *     coeff[t] (x)_{e in [site_start[t], site_start[t+1])} M_e,
 *     M_e[a, (a + shift[e]) mod d] = weight[e][a]  (zero elsewhere)
 * on qudit site[e]; a qudit no entry names carries the identity.  The sites of
 * one term are distinct. */
typedef struct pb200_op_terms {
    int32_t n_terms;
    const double*  coeff;       /* complex128 [n_terms] */
    const int32_t* site_start;  /* [n_terms + 1] into the per-site arrays */
    const int32_t* site;        /* qudit index k (0 = most significant digit) */
    const int32_t* shift;       /* m in [0, d) */
    const double*  weight;      /* complex128 [n_site_entries][d]: w_k[a] */
} pb200_op_terms;
/* out[c] = <psi_{traj0+c}| op |psi_{traj0+c}> as (re, im), not normalised,
 * matrix-free on the device.  A shard plan is refused (pb200_shards_expect),
 * as is a plan that carries a density matrix (PB200_ERR_UNSUPPORTED). */
int pb200_state_expect(pb200_plan* plan, int32_t traj0, int32_t count,
                       const pb200_op_terms* op, double* out);

/* Bitstring sampling on the device (QutipResult._weights + multinomial,
 * qutip_result.py:101-158, pulser/math/multinomial.py:17-36): weights over the
 * 2^N bitstrings (bit k = [digit_k == one_digit]), normalised, cumulated, and
 * searched with the caller's uniforms u[n_shots] (np.random.rand): out[i] =
 * bitstring index of shot i.  Only 8*n_shots bytes travel each way. */
int pb200_state_sample(pb200_plan* plan, int32_t traj, int32_t one_digit,
                       const double* uniforms, int32_t n_shots, int64_t* out);
/* Copy the current state of trajectory src_traj of `src` into trajectory dst_traj of `dst`, device to device
 * (same device, same Hilbert space).  Lets the observables of the generic backend evaluate <psi|H(t)|psi> with the
 * NOISELESS Hamiltonian (the operator qutip_backend.py:258-264 hands to every observable) on the state of a noisy
 * trajectory without a host round trip. */
int pb200_state_copy(pb200_plan* dst, int32_t dst_traj, pb200_plan* src, int32_t src_traj);
/* Device pointer of the current state buffer (complex128 [n_traj][D]). */
int pb200_state_device_ptr(pb200_plan* plan, void** dptr);

/* ---- density matrices ------------------------------------------------------ */
/* Reductions of the density matrices of a plan with a dissipator
 * (pb200_plan_set_dissipator): the plan holds vec(rho_b)[r*D + c] = rho_b[r, c]
 * for N = n_qudits / 2 physical qudits, D = dim^N.  They give the observables of
 * a master-equation run (default_observables.py:184-561 on a density matrix)
 * without copying rho to the host.  Values are NOT divided by the trace; the
 * caller normalises.  A plan without a dissipator is refused
 * (PB200_ERR_UNSUPPORTED).  On a shard of vec(rho) (one trajectory, holding the
 * rows [r0, r0 + D / G) of rho) each reduction returns the share of those rows,
 * read from the shard's own slice: the sum over the G shards is the value of the
 * whole matrix (pb200_density_sample: the shots of the shard's block of 2^N / G
 * bitstrings, out = their low N - shard_bits bits, as pb200_state_sample). */
/* trace[c] = Re Tr rho_{traj0+c} */
int pb200_density_trace(pb200_plan* plan, int32_t traj0, int32_t count,
                        double* trace);
/* occ[count][N]: occ[c][k] = sum_r rho_rr [digit_k(r) == digit] */
int pb200_density_occupation(pb200_plan* plan, int32_t traj0, int32_t count,
                             int32_t digit, double* occ);
/* corr[count][N][N] = Tr(n_i n_j rho), n_k = |digit><digit| on qudit k */
int pb200_density_correlation(pb200_plan* plan, int32_t traj0, int32_t count,
                              int32_t digit, double* corr);
/* out[c] = Tr(op rho_{traj0+c}) as (re, im), op as in pb200_state_expect;
 * term t reads rho[shift_t(r), r], one element per (term, r) (on a shard:
 * rho[r, shift_t(r)] of its own rows r). */
int pb200_density_expect(pb200_plan* plan, int32_t traj0, int32_t count,
                         const pb200_op_terms* op, double* out);
/* energy[c] = Re Tr(H rho_{traj0+c}), h2[c] = Re Tr(H^2 rho_{traj0+c}) with
 * H = H(t_us) of `ham`: a single-trajectory state-vector plan of the same
 * register and basis on the same device (the noiseless Hamiltonian handed to the
 * observables).  Reads the diagonal, the drive transitions and the interaction
 * diagonal of H: O(D (1 + N n_drives)^2) loads, never the whole matrix.  XY
 * registers are refused (PB200_ERR_UNSUPPORTED).  A shard sums Tr(rho H) and
 * Tr(rho H^2) over its own rows, with a `ham` plan on its own device. */
int pb200_density_energy(pb200_plan* plan, pb200_plan* ham, double t_us,
                         int32_t traj0, int32_t count, double* energy,
                         double* h2);
/* out[c] = <phi|rho_{traj0+c}|phi> as (re, im); phi: complex128[D] on the
 * host (Fidelity observable).  One pass over the D^2 entries. */
int pb200_density_overlap(pb200_plan* plan, int32_t traj0, int32_t count,
                          const double* phi, double* out);
/* Bitstring shots of trajectory `traj` drawn from diag(rho) with the recipe and
 * the caller's uniforms of pb200_state_sample (negative rounding noise on the
 * diagonal counts as 0). */
int pb200_density_sample(pb200_plan* plan, int32_t traj, int32_t one_digit,
                         const double* uniforms, int32_t n_shots, int64_t* out);

/* ---- hot path ------------------------------------------------------------ */
/* Advance every trajectory from t_start to t_stop (microseconds, inside the
 * sampling-time range).  Replaces the qutip.sesolve call at
 * simulation.py:729-735 for one [t_k, t_k+1] stretch of `tlist`. */
int pb200_propagate(pb200_plan* plan, double t_start, double t_stop,
                    const pb200_run_opts* opts, pb200_run_stats* stats);

/* out = H(t) * in for trajectory `traj`, host buffers of D complex numbers.
 * Replaces QobjEvo.__call__(t) @ psi, i.e. get_hamiltonian(t)
 * (simulation.py:625-661) applied to a vector. */
int pb200_apply_h(pb200_plan* plan, int32_t traj, double t_us,
                  const double* in, double* out);

/* Interpolated coefficient of (drive, row) at time t: out[0..1] = coef (re,im),
 * out[2] = det.  The QobjEvo coefficient interpolant itself. */
int pb200_coefficients_at(pb200_plan* plan, int32_t traj, int32_t drive,
                          int32_t row, double t_us, double* out3);

/* Time the bare H-apply kernel: `reps` applies of H(t) on the resident state,
 * device time in ms through CUDA events (roofline measurement). */
int pb200_bench_apply(pb200_plan* plan, double t_us, int32_t reps,
                      double* ms_out, int64_t* launches_out);

/* ---- state-vector shards (registers larger than one GPU) -------------------- */
/* Shard `shard_index` of G = 2^shard_bits (shard_bits = 1, 2, 3) of ONE state
 * of desc->n_qudits = N qubits: the plan holds the global indices
 * [i 2^L, (i+1) 2^L), L = N - shard_bits (13 <= L <= 29), i.e. the top
 * shard_bits qubits (qudits 0 .. shard_bits-1) select the shard.  d = 2, one
 * drive, n_traj = 1.  Uploads (interaction, drive) are those of a whole plan;
 * each shard computes its slice of the interaction diagonal.  A shard answers
 * pb200_state_set (basis_index: the global index; psi: its slice), _get,
 * _probabilities, _norm2, _overlap (phi: its slice) and _sample (out: the low L
 * bits of the bitstring) on its slice, and _occupation / _correlation with its
 * contributions (global digits); pb200_propagate / _apply_h / _state_energy
 * fail with PB200_ERR_STATE: use the group calls below.  Argument checks
 * happen before any device call. */
int pb200_plan_create_shard(pb200_plan** out, const pb200_plan_desc* desc,
                            int32_t shard_bits, int32_t shard_index);
/* Link the G shards plans[i] = shard i (after their uploads): checks N, sampling
 * times and the Taylor structure (one global drive, of any phase; vec(rho):
 * one phase, the same dissipator on every shard), merges the interaction bounds
 * so that every shard schedules exactly like the unsharded plan, enables peer
 * access between distinct devices (PB200_ERR_UNSUPPORTED where it is
 * impossible). */
int pb200_shards_link(pb200_plan** plans, int32_t count);
/* pb200_propagate of the whole state with the Taylor propagator (integrator 0
 * or 3; options steering the Magnus controller are refused): the schedule is
 * computed once, each order of the series runs on every shard, reading the
 * peers' slices across the shard bits. */
int pb200_shards_propagate(pb200_plan** plans, int32_t count, double t_start,
                           double t_stop, const pb200_run_opts* opts,
                           pb200_run_stats* stats);
/* out = H(t) in, host buffers of the FULL 2^N complex amplitudes. */
int pb200_shards_apply_h(pb200_plan** plans, int32_t count, double t_us,
                         const double* in, double* out);
/* <psi|H(t)|psi> and <psi|H(t)^2|psi> of the sharded state (energy[1], h2[1]). */
int pb200_shards_energy(pb200_plan** plans, int32_t count, double t_us,
                        double* energy, double* h2);
/* <psi| op |psi> of the sharded state, out[2] = (re, im), not normalised.  A
 * term that changes shard bits x reads shard r ^ x from shard r: peer access
 * between the devices of every such pair is enabled here when missing
 * (PB200_ERR_UNSUPPORTED where there is none). */
int pb200_shards_expect(pb200_plan** plans, int32_t count,
                        const pb200_op_terms* op, double* out);

/* ---- host-side math, usable without a device (exercised by the CPU tests) -- */
/* Interpolant of complex samples y[n] (re,im) over x[n] at nq query points:
 * out[nq][2].  The QobjEvo array-coefficient rule (order 0 / 1 / 3). */
int pb200_host_interpolate(const double* x, const double* y, int32_t n,
                           int32_t order, const double* tq, int32_t nq,
                           double* out);
/* Exact Magnus moments over [a, b] of the same interpolant:
 * out[0..1] = B0 = int S dt, out[2..3] = B1 = (1/(b-a)) int (t - (a+b)/2) S dt */
int pb200_host_moments(const double* x, const double* y, int32_t n,
                       int32_t order, double a, double b, double* out4);
/* Time-dependent Taylor propagator (integrator 3), host side.  Degree-p
 * polynomial in u = (t-a)/h, u in [0,1], of the same interpolant of REAL samples
 * y[n] on [a, a+h] (Chebyshev interpolation): coeffs[p+1] monomial coefficients,
 * *resid = max |polynomial - interpolant| on the step.  p <= 8. */
int pb200_host_taylor_fit(const double* x, const double* y, int32_t n,
                          int32_t order, double a, double h, int32_t p,
                          double* coeffs, double* resid);
/* Separable structure of a batch of drive tables (what lets noise-trajectory
 * batches run on integrator 3): coef[n_traj][n_qudits][n_times] (re,im) and
 * det[n_traj][n_qudits][n_times] as handed to pb200_plan_set_drive (rows = N).
 * *separable = 1 when coef_{b,k} = a_{b,k} * (largest drive row) and
 * det_{b,k} = det_{0,0} + c_{b,k} * m with one common shape m (max |m| = 1), to
 * 2e-13 of the largest sample; then a_out[n_traj][n_qudits] (re,im),
 * c_out[n_traj][n_qudits], m_out[n_times] (any may be NULL).  Restates what
 * HamiltonianData._sample_with_trajectory does to Global samples
 * (pulser-core/pulser/_hamiltonian_data/hamiltonian_data.py:408-534): amp *=
 * fluctuation * waist factor, det += doppler shift inside the pulse slots. */
int pb200_host_taylor_separable(const double* coef, const double* det,
                                int32_t n_traj, int32_t n_qudits,
                                int32_t n_times, int32_t* separable,
                                double* a_out, double* c_out, double* m_out);
/* Separable structure with several detuning time shapes (what lets detuning-map
 * sequences, masks and their noisy batches run on integrator 3): same tables
 * and drive factors as pb200_host_taylor_separable, with
 * det_{b,k} = det_{0,0} + sum_{s < S} c_{b,k,s} * m_s, each max |m_s| = 1, to
 * 2e-13 of the largest sample, S <= max_shapes <= 4.  Pulser's detuning map
 * modulator adds -w_k eps(t) n_k to every atom k
 * (pulser-core/pulser/sampler/samples.py:560-601): one shape per map.
 * *n_shapes = S, or -1 when the drive rows are not multiples of one row or the
 * detuning needs more than max_shapes shapes; then a_out[n_traj][n_qudits]
 * (re,im), c_out[n_traj][n_qudits][max_shapes], m_out[max_shapes][n_times]
 * (unused shapes 0; any may be NULL). */
int pb200_host_taylor_shapes(const double* coef, const double* det,
                             int32_t n_traj, int32_t n_qudits, int32_t n_times,
                             int32_t max_shapes, int32_t* n_shapes,
                             double* a_out, double* c_out, double* m_out);
/* Order K of the Taylor series of a step of length h whose generator obeys
 * |H_j| <= m[j] (j = 0..p): smallest K with remainder bound *tail_out <= tol. */
int pb200_host_taylor_order(double h, const double* m, int32_t p, double tol,
                            int32_t* order_out, double* tail_out);
/* First order k_lo of such a step of K orders whose outputs may be stored in
 * single precision (g_stored: the step stores G_k = X chi_k as well): the
 * smallest k_lo whose bound on the rounding's effect on psi(a+h),
 * *bound_out, is <= tol (K when none is). */
int pb200_host_taylor_lowprec(double h, const double* m, int32_t p, int32_t K,
                              int32_t g_stored, double tol, int32_t* k_lo_out,
                              double* bound_out);
/* Chebyshev coefficients a_j of exp(-i*rho*x) on [-1,1], truncated at tol:
 * writes up to cap (re,im) pairs, returns the count through *count. */
int pb200_host_chebyshev(double rho, double tol, double* out, int32_t cap,
                         int32_t* count);

#ifdef __cplusplus
}
#endif
#endif /* PULSER_B200_H */
