"""CPU: pins the oracle's centre-surround model with a float32 photoreceptor state (cutoff_hz = 0) against fixtures the
unmodified reference produced (oracle/make_golden_cs32.py): rows in order, counters, cs_steps_taken and the final lp,
base and surround, bit for bit. At cutoff_hz = 0 low_pass_filter returns the float32 log frame (emulator_utils.py:75-77)
and the surround is its clone (emulator.py:1063), so every op of the Euler step is float32 -- unlike the float64 state,
whose p_term and change are float64. The sensitivity tests show the fixtures tell the two rules apart."""
import functools

import numpy as np
import pytest

from emu_oracle_cs32 import OracleEmulatorCS32, lib
from helpers import TapeRNG, assert_events_equal, canonical, load_golden, split_events

CS32_GOLDENS = ["emu_cs32_120x176", "emu_cs32_37x53", "emu_cs32_scidvs", "emu_cs32_clean"]


@functools.lru_cache(maxsize=None)
def run_oracle(name, f64_rule=0, alpha_h_ulps=0):
    g = load_golden(name)
    rng = TapeRNG(g["tape"])
    L = lib()
    L.oracle_set_cs_f64_rule(f64_rule)
    L.oracle_set_cs_perturbation(0, alpha_h_ulps)
    try:
        em = OracleEmulatorCS32(rng=rng, **g["kwargs"])
        if "dvs_params" in g:
            em.set_dvs_params(str(g["dvs_params"]))
        rows = [em.generate_events(f, float(t)) for f, t in zip(g["frames"], g["times"])]
    finally:
        L.oracle_set_cs_f64_rule(0)
        L.oracle_set_cs_perturbation(0, 0)
    return dict(rows=rows, steps=list(em.cs_steps_taken), on=em.num_events_on, off=em.num_events_off,
                exhausted=rng.exhausted(), lp=em.lp, base=em.base, surround=em.surround)


@pytest.mark.parametrize("name", CS32_GOLDENS)
def test_oracle_matches_reference_golden_f32(name):
    g = load_golden(name)
    got = run_oracle(name)
    want = split_events(g["events"], g["event_counts"])
    for i, w in enumerate(want):
        assert_events_equal(got["rows"][i], w, exact_order=True, ctx="%s frame %d" % (name, i))
    assert got["exhausted"]
    assert got["on"] == int(g["num_on"]) and got["off"] == int(g["num_off"])
    assert got["steps"] == list(g["cs_steps_taken"])
    for key in ("lp", "base", "surround"):
        ref = g["state_%s" % {"lp": "lp_log_frame", "base": "base_log_frame", "surround": "cs_surround_frame"}[key]]
        assert ref.dtype == np.float32 and got[key].dtype == np.float32, key
        assert np.array_equal(got[key].view(np.uint32), ref.view(np.uint32)), key


@pytest.mark.parametrize("name", ["emu_csdvs", "emu_csdvs_37x53"])
def test_float64_state_is_emu_oracle_c(name):
    """The float32 oracle library hands a float64 state to emu_oracle.c: the float64 centre-surround fixtures come out
    as they do there."""
    g = load_golden(name)
    rng = TapeRNG(g["tape"])
    em = OracleEmulatorCS32(rng=rng, **g["kwargs"])
    want = split_events(g["events"], g["event_counts"])
    for i, (f, t) in enumerate(zip(g["frames"], g["times"])):
        assert_events_equal(em.generate_events(f, float(t)), want[i], exact_order=True, ctx="%s frame %d" % (name, i))
    assert em.cs_steps_taken == list(g["cs_steps_taken"])
    assert em.surround.dtype == np.float64 and np.array_equal(em.surround, g["state_cs_surround_frame"])


def test_fixtures_pin_early_stop_and_full_count():
    """Every fixture has a frame whose iteration stops before num_steps (the uniform pair: one step) and frames that run
    all their steps."""
    import math
    for name in CS32_GOLDENS:
        g = load_golden(name)
        k = g["kwargs"]
        tau_p = k["cs_tau_p_ms"] * 1e-3
        tau_h = tau_p / k["cs_lambda_pixels"] ** 2
        dts = np.diff(g["times"])
        planned = [int(math.ceil((dt / min(tau_p, tau_h)) * 5)) for dt in dts]
        taken = list(g["cs_steps_taken"])
        assert any(t < p for t, p in zip(taken, planned)), (name, taken, planned)
        assert any(t == p for t, p in zip(taken, planned)), (name, taken, planned)


def _differences(got, want):
    rows = 0
    for g, w in zip(got["rows"], want["rows"]):
        g, w = canonical(g), canonical(w)
        rows += int((g != w).any(axis=1).sum()) if g.shape == w.shape else abs(len(g) - len(w)) + min(len(g), len(w))
    return rows, int((got["surround"].view(np.uint32) != want["surround"].view(np.uint32)).sum())


@pytest.mark.parametrize("perturbation", [dict(f64_rule=1), dict(f64_rule=2), dict(alpha_h_ulps=1)],
                         ids=["p_term_f64", "change_f64", "alpha_h_1ulp"])
def test_perturbed_rule_is_caught(perturbation):
    """The float64 state's rule (p_term, or the sum change, in float64) or alpha_h one ulp up must move the rows or
    the surround of at least one fixture."""
    total_rows = total_px = 0
    for name in CS32_GOLDENS:
        rows, px = _differences(run_oracle(name, **perturbation), run_oracle(name))
        print("%s %s: %d rows and %d surround pixels differ" % (name, perturbation, rows, px))
        total_rows += rows
        total_px += px
    assert total_rows + total_px > 0
