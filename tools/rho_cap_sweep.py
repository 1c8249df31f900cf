"""Sweep of the Chebyshev half-width cap and the longest Magnus step (VERDICT r01 item 1).

For every (PB200_RHO_CAP_MILLI, max_step_samples):
  (i)   error against the DOP853 oracle at N = 10 / 12 on the C2 shape,
  (ii)  self-convergence against a tol = 1e-11 run at N = 20,
  (iii) H-applies per ns and time-steps/s at N = 20.
Writes one JSON line per case to stdout.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

from pulser_b200 import engine, workloads as W
from oracle import evolve
from oracle.ref_hamiltonian import OracleHamiltonian

CAPS = [int(x) for x in os.environ.get("SWEEP_CAPS", "3600,6000,12000,24000,48000").split(",")]
KS = [int(x) for x in os.environ.get("SWEEP_KS", "32,64,128").split(",")]
SMALL = [int(x) for x in os.environ.get("SWEEP_SMALL", "10,12").split(",")]
BIG = int(os.environ.get("SWEEP_BIG", "20"))


def run(plan, tf, **kw):
    plan.set_state("all-ground")
    t0 = time.perf_counter()
    st = plan.propagate(0.0, tf, **kw)
    wall = time.perf_counter() - t0
    return st, wall


def main():
    refs = {}
    for n in SMALL:
        spec = W.config_c2(n=n)
        psi0 = evolve.all_ground_state(spec)
        tf = spec.sampling_times[-1]
        refs[n] = evolve.sesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-13, atol=1e-15)[-1]
    spec_big = W.config_c2(n=BIG)
    tfb = spec_big.sampling_times[-1]
    with engine.DevicePlan(spec_big) as pb:
        os.environ["PB200_RHO_CAP_MILLI"] = "3600"
        run(pb, tfb)  # warm-up
        st, wall = run(pb, tfb, tol=1e-11)
        ref_big = pb.get_state()[0]
        print(json.dumps({"case": "reference_run_tol1e-11", "n": BIG, "applies_per_ns": st["n_applies"] / 4000,
                          "gpu_ms": st["gpu_ms"]}), flush=True)
        for integ in (1, 2):
            for cap in CAPS:
                for K in KS:
                    os.environ["PB200_RHO_CAP_MILLI"] = str(cap)
                    os.environ["PB200_RHO_CAP_KRYLOV_MILLI"] = str(max(cap, 12000))
                    row = {"integrator": integ, "cap": cap * 1e-3, "K": K}
                    for n in SMALL:
                        spec = W.config_c2(n=n)
                        with engine.DevicePlan(spec) as p:
                            st, _ = run(p, spec.sampling_times[-1], max_step=K, integrator=integ)
                            got = p.get_state()[0]
                        row[f"err_n{n}"] = float(np.linalg.norm(got - refs[n]))
                        row[f"applies_per_ns_n{n}"] = st["n_applies"] / 4000
                    st, wall = run(pb, tfb, max_step=K, integrator=integ)
                    got = pb.get_state()[0]
                    row.update({
                        "n": BIG, "self_err": float(np.linalg.norm(got - ref_big)),
                        "applies_per_ns": st["n_applies"] / 4000, "steps_per_s": 4000 / (st["gpu_ms"] * 1e-3),
                        "wall_steps_per_s": 4000 / wall, "mean_step": st["mean_step_samples"],
                        "n_steps": st["n_steps"], "n_checks": st["n_checks"], "max_rho": st["max_rho"],
                        "us_per_apply": st["gpu_ms"] * 1e3 / max(st["n_applies"], 1),
                        "err_estimate": st["err_estimate"], "launches": st["n_launches"],
                    })
                    print(json.dumps(row), flush=True)


main()
