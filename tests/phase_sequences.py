"""Pulser sequences whose global drive phase changes in time (needs pulser-core): two pulses of different phase, a
`phase_shift` between pulses, and an EOM block with phase-drift correction."""
from __future__ import annotations

import numpy as np

from pulser_b200 import workloads as W

KINDS = ("phases", "phase_shift", "eom")


def phase_sequence(kind: str, n: int = 13):
    """`phases` / `phase_shift` use smooth interpolated amplitudes, which the auto rule hands to the Taylor
    propagator (a 200 ns Blackman on the 1 ns grid is too curved for multi-interval steps at the default tolerance,
    whatever its phase); `eom` is a square-pulse EOM block on AnalogDevice"""
    import pulser
    from pulser.waveforms import ConstantWaveform, InterpolatedWaveform, RampWaveform

    reg = pulser.Register.from_coordinates(W.disc_register(n, 14.0, 6.0, n), prefix="q")
    if kind == "eom":
        seq = pulser.Sequence(reg, pulser.AnalogDevice)
        seq.declare_channel("ryd", "rydberg_global")
        seq.enable_eom_mode("ryd", amp_on=3.0, detuning_on=0.0, optimal_detuning_off=-2.0, correct_phase_drift=True)
        seq.add_eom_pulse("ryd", 100, phase=0.0, correct_phase_drift=True)
        seq.delay(100, "ryd")
        seq.add_eom_pulse("ryd", 100, phase=0.5, correct_phase_drift=True)
        seq.disable_eom_mode("ryd", correct_phase_drift=True)
        return seq
    seq = pulser.Sequence(reg, pulser.MockDevice)
    seq.declare_channel("ryd", "rydberg_global")

    def amp():
        return InterpolatedWaveform(200, [0.0, 4.0, 8.0, 8.0, 4.0, 0.0])

    seq.add(pulser.Pulse(amp(), ConstantWaveform(200, -1.0), 0.0), "ryd")
    if kind == "phases":
        seq.add(pulser.Pulse(ConstantWaveform(150, 0.0), ConstantWaveform(150, -1.0), 0.0), "ryd")
        seq.add(pulser.Pulse(amp(), RampWaveform(200, -1.0, 2.0), 1.3), "ryd")
    elif kind == "phase_shift":
        seq.phase_shift(0.9, *reg.qubit_ids, basis="ground-rydberg")
        seq.add(pulser.Pulse(amp(), RampWaveform(200, -1.0, 2.0), 0.0), "ryd")
    else:
        raise ValueError(kind)
    return seq


def moving_phase_rows(spec) -> bool:
    """the drive rows are identical (one global drive), and their phase where the amplitude is non-zero moves"""
    coef = np.asarray(spec.drives[0].coef)
    assert len(spec.drives) == 1 and (coef == coef[:1]).all()
    row = coef[0]
    on = np.abs(row) > 1e-9 * np.abs(row).max()
    ph = np.angle(row[on] / row[on][np.argmax(np.abs(row[on]))])
    return bool(np.ptp(ph) > 1e-3)
