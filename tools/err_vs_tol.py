import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from pulser_b200 import engine, workloads as W
from oracle import evolve
from oracle.ref_hamiltonian import OracleHamiltonian
integ = int(os.environ.get("INTEG", "1"))
for n in (8, 11):
    spec = W.config_c2(n=n, seed=20)
    psi0 = evolve.all_ground_state(spec); tf = spec.sampling_times[-1]
    ref = evolve.sesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-13, atol=1e-15)[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf, integrator=integ)
        got = plan.get_state()[0]
        print(json.dumps({"n": n, "integ": integ, "err2": float(np.linalg.norm(got-ref)), "mean_step": round(st["mean_step_samples"],2),
                          "applies_per_ns": round(st["n_applies"]/4000,2)}))
