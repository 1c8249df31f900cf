"""Experiment (GPU): what the observables of a master-equation run cost through ``B200Backend``, with the density
matrices left on the device (``DeviceDensityView``, the streamed path) and with every density matrix downloaded and
replayed on the host (the path the backend takes when the plan has no density reductions).

Case: C2's blockade sweep (SURVEY 8d) shortened to 50 / 200 / 50 ns as in ``experiments/lindblad_cost.py``, as a pulser
Sequence on MockDevice's global Rydberg channel over C2's disc registers of N = 10, 12, 13 atoms, with dephasing 0.05
and relaxation 0.01 rad/us, and ``Occupation``, ``CorrelationMatrix``, ``Energy`` and ``EnergyVariance`` at 21
evaluation times.  Each (N, path) runs in a fresh process, so its peak host RSS is its own.  Reported: wall time of the
run, split into propagation (every ``LindbladPlan.propagate`` call, which returns once the device is done) and the rest
(observables, and for the replay the downloads of the stored density matrices), peak host RSS, and the card's memory
in use after the run (the buffer pool keeps what the plans took, so it bounds the peak).  The replay runs only where
its stored density matrices (21 x 16 x 4^N bytes) fit twice in the host's available memory; otherwise the case records
why it was skipped.  The card name and power limit are read in the same run.  Prints one JSON object.

Usage: python experiments/density_observables_cost.py [--sizes 10,12,13] [--timeout S] [--out FILE]
"""
from __future__ import annotations

import json
import os
import resource
import subprocess
import sys
import time
import warnings

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
N_TIMES = 21


def sequence(n: int):
    import pulser_b200.backend  # noqa: F401  (makes pulser-core importable)
    import pulser
    from pulser.waveforms import ConstantWaveform, RampWaveform

    from pulser_b200 import workloads as W

    omega = 2 * np.pi * 1.5
    d0, df = -3 * omega, omega  # W.blockade_sweep_waveforms: -6 U and 2 U with U = omega / 2
    coords = W.disc_register(n, 38.0, 5.0, n)
    seq = pulser.Sequence(pulser.Register.from_coordinates(coords, prefix="q"), pulser.MockDevice)
    seq.declare_channel("ryd", "rydberg_global")
    seq.add(pulser.Pulse(RampWaveform(50, 0.0, omega), ConstantWaveform(50, d0), 0.0), "ryd")
    seq.add(pulser.Pulse(ConstantWaveform(200, omega), RampWaveform(200, d0, df), 0.0), "ryd")
    seq.add(pulser.Pulse(RampWaveform(50, omega, 0.0), ConstantWaveform(50, df), 0.0), "ryd")
    return seq


def run_case(n: int, path: str) -> dict:
    import pulser_b200.backend  # noqa: F401  (makes pulser-core importable)
    import pulser
    import torch
    from pulser.backend.default_observables import CorrelationMatrix, Energy, EnergyVariance, Occupation

    from pulser_b200 import B200Backend, B200Config, lindblad

    prop = {"s": 0.0, "calls": 0}
    orig = lindblad.LindbladPlan.propagate

    def timed(self, *a, **k):
        t0 = time.perf_counter()
        try:
            return orig(self, *a, **k)
        finally:
            prop["s"] += time.perf_counter() - t0
            prop["calls"] += 1

    lindblad.LindbladPlan.propagate = timed
    times = list(np.linspace(0.0, 1.0, N_TIMES))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cfg = B200Config(observables=[Occupation(evaluation_times=times), CorrelationMatrix(evaluation_times=times),
                                      Energy(evaluation_times=times), EnergyVariance(evaluation_times=times)],
                         noise_model=pulser.NoiseModel(dephasing_rate=0.05, relaxation_rate=0.01))
        be = B200Backend(sequence(n), config=cfg)
        assert be._streams_density()
        if path == "replay":
            be._streams_density = lambda: False
        t0 = time.perf_counter()
        res = be.run()
        wall = time.perf_counter() - t0
    free, total = torch.cuda.mem_get_info()
    return {
        "n": n, "path": path, "wall_s": wall, "propagation_s": prop["s"], "observables_s": wall - prop["s"],
        "propagate_calls": prop["calls"],
        "peak_host_rss_gib": resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20,
        "device_mem_in_use_gib": (total - free) / 2**30,
        "final_occupation": [float(x) for x in np.real(res.get_result("occupation", 1.0))],
        "final_energy": float(np.real(res.get_result("energy", 1.0))),
        "final_energy_variance": float(np.real(res.get_result("energy_variance", 1.0))),
    }


def mem_available() -> int:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    raise RuntimeError("MemAvailable missing from /proc/meminfo")


def main() -> None:
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="10,12,13")
    ap.add_argument("--case", default=None, help="internal: N,path of one case")
    ap.add_argument("--timeout", type=float, default=900.0, help="seconds per case")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.case:
        n, path = args.case.split(",")
        print(json.dumps(run_case(int(n), path)))
        return
    from experiments.shard_scaling import gpu_info

    out = {"gpu": gpu_info(), "n_times": N_TIMES, "cases": []}
    for n in [int(x) for x in args.sizes.split(",")]:
        for path in ("streamed", "replay"):
            stored = N_TIMES * 16 * 4**n
            if path == "replay" and 2 * stored > mem_available():
                case = {"n": n, "path": path, "skipped": f"the stored density matrices need {stored / 2**30:.1f} GiB, "
                        f"the host has {mem_available() / 2**30:.1f} GiB available"}
            else:
                try:
                    p = subprocess.run([sys.executable, os.path.abspath(__file__), "--case", f"{n},{path}"],
                                       capture_output=True, text=True, timeout=args.timeout)
                except subprocess.TimeoutExpired:
                    p = None
                if p is None:
                    case = {"n": n, "path": path, "skipped": f"did not finish within {args.timeout} s"}
                elif p.returncode != 0:
                    case = {"n": n, "path": path, "failed": p.stderr[-2000:]}
                else:
                    case = json.loads(p.stdout.strip().splitlines()[-1])
            out["cases"].append(case)
            print(json.dumps(case), flush=True)
    text = json.dumps(out)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
