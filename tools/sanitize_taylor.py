"""compute-sanitizer target: the Taylor stage kernels on short sequences (uniform N = 12 and 5; a 3-trajectory noise batch
at N = 11: per-trajectory table in shared memory, blockIdx.y = trajectory)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from pulser_b200 import engine, workloads as W

amp, det = W.blockade_sweep_waveforms(t_rise=40, t_sweep=80, t_fall=40)
for n in (12, 5):
    spec = W.ising_global_spec(W.disc_register(n, 16.0, 5.0, 3), W.C6_LEVEL_60, amp, det, phase=0.3 if n == 5 else 0.0)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1], integrator=3)
        print("uniform n", n, "launches", st["n_launches"], "norm2", float(plan.norm2()[0]))
n = 11
coords = W.disc_register(n, 14.0, 5.0, 5)
base = W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det)
rng = np.random.default_rng(1)
specs = [W.noisy_trajectory_spec(base, coords, rng.normal(0, 1.5, n), 1.03, 60.0) for _ in range(3)]
with engine.DevicePlan(specs) as plan:
    plan.set_state("all-ground")
    st = plan.propagate(0.0, base.sampling_times[-1])
    print("batch n", n, "integrator", st["integrator"], "launches", st["n_launches"], "norm2", plan.norm2())
# master equation (DISS kernels): N = 3 (small kernel, 2N = 6) and N = 7 (tiled, both-flip partners in and above the tile)
from pulser_b200.lindblad import LindbladPlan
ops = np.array([np.diag([np.sqrt(0.1), 0.0]), [[0.0, 0.0], [0.3, 0.0]]], dtype=complex)
for n in (3, 7):
    spec = W.ising_global_spec(W.disc_register(n, 16.0, 5.0, 3), W.C6_LEVEL_60, amp, det)
    spec.collapse_ops = ops
    with LindbladPlan(spec) as lp:
        lp.set_state(np.eye(1, 2**n, 2**n - 1)[0])
        st = lp.propagate(0.0, spec.sampling_times[-1], integrator=3)
        print("lindblad n", n, "launches", st["n_launches"], "trace", np.trace(lp.get_rho()[0]).real)
# master equation under a moving drive phase (CPLX + DISS kernels): a phase jump of pi/2 mid-sweep, N = 3 (small kernel)
# and N = 7 (tiled)
ph = np.where(np.arange(len(amp)) < len(amp) // 2, 0.0, np.pi / 2)
for n in (3, 7):
    spec = W.ising_global_spec(W.disc_register(n, 16.0, 5.0, 3), W.C6_LEVEL_60, amp, det, phase=ph)
    spec.collapse_ops = ops
    with LindbladPlan(spec) as lp:
        lp.set_state(np.eye(1, 2**n, 2**n - 1)[0])
        st = lp.propagate(0.0, spec.sampling_times[-1], integrator=3)
        print("lindblad phase jump n", n, "launches", st["n_launches"], "trace", np.trace(lp.get_rho()[0]).real)
