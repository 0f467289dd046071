"""The device's numpy noise stream (k_md.cuh ``md_refnoise_cta``) on the window-scheme paths that natural draws reach
rarely or never: planted draws on numpy's own tables, and stress tables, against the sequential ziggurat.

The kernel does not run numpy's sequential algorithm but a parallel window scheme (DESIGN §7): windows of
``refnoise.window_size`` draws cut into per-thread chunks, an ordered list of at most ``NZ_LIST`` non-fast positions
(a window holding more stops at the first it cannot list), anchor runs that mark the draws consumed inside slow and
tail attempts, a prefix count that numbers the normals, and another window when one yields too few.  Natural streams
never overflow the list (a full window holds ~490 non-fast positions), never leave an uncapped window short, and only
a capped window can have a consumed attempt straddle its end.  Every case here reaches such a path in its first step:

* planted draws: a state whose XSL-RR output is a chosen raw value, stepped back so that the value lands at a chosen
  draw of the step.  The stream is a genuine PCG64 stream, so the oracle is ``np.random.Generator`` itself.
* stress tables: ``ki`` / ``fi`` / ``wi`` edited so slow attempts, rejections or long tails are common.  The oracle is
  the sequential restatement ``refnoise.normals_from_raw`` with the same tables.

Every step checks the device's PCG64 state exactly and its normals bit for bit (idx-0 tail values within 2 ulp: the
device's ``log1p`` is not glibc's).  Before any launch the host checks that no consumed slow or tail decision lies
within 4 ulp of its threshold (so a device ``exp`` / ``log1p`` last-bit difference cannot flip it) and bounds every step
to at most 128 windows and 32 tail rounds at every position the device classifies.

Measured on one H100 80GB HBM3 (700 W power limit): all 15 cases equal the sequential stream in every step, state and
normals.  First-step events (m normals per step):

  cap{10005,5500}_tail_at_window_end  m 60,030 / 33,000: a 3-round tail planted at draw 32,767 of the capped first
                                      window is consumed; the second window starts past W
  cap{10005,5500}_slow_at_window_end  the same with an accepted slow attempt
  p1_tail_at_{first_draw,window_end}  m 6 (W 71, T 18, C 4): 3-round tails at draw 0 (consumed) and draw 70 (classified)
  c{4,5,32}_tail_on_chunk_end         m 3,912 / 3,918 / 60,030: a 3-round tail on a chunk's last draw, 2 tails
                                      straddle a chunk boundary
  crowded_m60030                      6 windows, 3 capped, 4 list cuts, 2 short
  all_slow_m996 / all_slow_m6000      4 windows, 1 cut, 3 short / 14 windows, 10 cuts, 13 short, 2 restarts past W
  rejecting_m996                      8 windows, no cut, 7 short
  long_tails_m6 / long_tails_m12000   a 4-round tail planted at draw 3 (C 4) / C 13, 7 straddling tails, 8 rounds

Of 478 tail values over all steps, 5 differed, each by 1 ulp (long_tails_m12000); every other normal was
bit-identical.  The GPU tests of this file took 16.6 s, 3.1 s of it the host plans.  The cases have teeth: a kernel
that restarts the next window at ``weff`` instead of ``max(cur, weff)`` fails the four cap*_at_window_end cases, both
all-slow cases and rejecting_m996; one that ignores the list cut fails crowded_m60030 and both all-slow cases; one
that counts a tail's draws only up to the window end fails both cap*_tail_at_window_end cases -- each at the first
step's state.
"""
import functools
import math
import os
import re
import time
from dataclasses import dataclass

import numpy as np
import pytest
import torch

from ai2bmd_b200 import refnoise as R
from ai2bmd_b200.engine import Engine
from ai2bmd_b200.fixtures import load_fragments
from ai2bmd_b200.md import FS, KB, MASSES

KT = 300.0 * KB
M64 = (1 << 64) - 1
MAX_WINDOWS, MAX_ROUNDS, MIN_ULPS = 128, 32, 4
K_MD = os.path.join(os.path.dirname(__file__), "..", "ai2bmd_b200", "csrc", "k_md.cuh")


# ---- tables ------------------------------------------------------------------------------------------------------
def _table(kind):
    """numpy's tables, or a stress edit of them; ``r`` is what the device derives it from, wi[255] * 2^52."""
    real = R.tables()
    if kind == "real":
        return real
    t = {k: np.array(real[k], copy=True) for k in ("wi", "ki", "fi")}
    if kind == "crowded":            # layers 1-16 always slow: ~6 % of draws, capped windows overflow the list
        t["ki"][1:17] = 0
    elif kind == "all-slow":         # every layer but 0 slow: every chunk boundary straddled, lists cut, windows short
        t["ki"][1:] = 0
    elif kind == "rejecting":        # layers 129-255 slow and always rejected: short windows without a cut
        t["ki"][128:] = 0
        t["fi"][128:] = 1.0
    elif kind == "long-tails":       # every idx-0 draw starts a tail, and r = 1.28 (not 3.65) rejects more rounds
        t["ki"][0] = 0
        t["wi"][255] *= 0.35
    else:
        raise ValueError(kind)
    t["r"] = float(t["wi"][255] * 2.0 ** 52)
    return t


# ---- cases -------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Case:
    table: str
    P: int                     # protein atoms: m = 6 P normals per step
    seed: int
    steps: int
    event: str                 # census entry the first step must reach
    at_least: int = 1
    plant: tuple = ()          # ("tail" | "slow", draw of the first step)


CASES = {
    # numpy's tables, planted draws: the oracle is Generator.standard_normal
    "cap10005_tail_at_window_end": Case("real", 10005, 11, 4, "tail_end_straddle", plant=("tail", 32767)),
    "cap5500_tail_at_window_end": Case("real", 5500, 12, 4, "tail_end_straddle", plant=("tail", 32767)),
    "cap10005_slow_at_window_end": Case("real", 10005, 13, 3, "slow_end_straddle", plant=("slow", 32767)),
    "cap5500_slow_at_window_end": Case("real", 5500, 14, 3, "slow_end_straddle", plant=("slow", 32767)),
    "p1_tail_at_first_draw": Case("real", 1, 15, 8, "planted_consumed", plant=("tail", 0)),
    "p1_tail_at_window_end": Case("real", 1, 16, 8, "planted_live", plant=("tail", 70)),
    "c4_tail_on_chunk_end": Case("real", 652, 17, 5, "tail_chunk_straddle", plant=("tail", 1999)),
    "c5_tail_on_chunk_end": Case("real", 653, 18, 5, "tail_chunk_straddle", plant=("tail", 1999)),
    "c32_tail_on_chunk_end": Case("real", 10005, 19, 3, "tail_chunk_straddle", plant=("tail", 16383)),
    # stress tables: the oracle is the sequential restatement on the same tables
    "crowded_m60030": Case("crowded", 10005, 1, 3, "cuts", 2),
    "all_slow_m996": Case("all-slow", 166, 1, 6, "short_uncapped"),
    "all_slow_m6000": Case("all-slow", 1000, 1, 4, "cuts", 5),
    "rejecting_m996": Case("rejecting", 166, 1, 6, "short_uncapped"),
    "long_tails_m6": Case("long-tails", 1, 21, 8, "tail_chunk_straddle", plant=("tail", 3)),
    "long_tails_m12000": Case("long-tails", 2000, 71, 4, "max_tail_rounds", 8),
}
# the first window's (W, T, C) for each protein size above: every regime of the window shape
SHAPES = {1: (71, 18, 4), 166: (1090, 273, 4), 652: (4094, 1024, 4), 653: (4100, 1024, 5), 1000: (6244, 1024, 7),
          2000: (12424, 1024, 13), 5500: (32768, 1024, 32), 10005: (32768, 1024, 32)}


def _rotl(v, k):
    return ((v << k) | (v >> (64 - k))) & M64 if k else v


def _planted_raw(tab, rng, kind):
    """A raw draw whose attempt is an idx-0 tail start or a slow (idx > 0, rabs >= ki) attempt."""
    i = 0 if kind == "tail" else int(rng.integers(1, 256))
    rabs = int(rng.integers(int(tab["ki"][i]), 1 << 52))
    return i | (int(rng.integers(0, 2)) << 8) | (rabs << 9)


def _plant(tab, inc, p, kind, rng):
    """A PCG64 state whose draw p is a planted attempt that is a live start: a tail of at least 3 rounds, or an accepted
    slow attempt.  The state S whose XSL-RR output is the value is any hi with lo = hi ^ rotl(value, hi >> 58); the
    step's state is S stepped back by p + 1."""
    for _ in range(20000):
        value = _planted_raw(tab, rng, kind)
        hi = int(rng.integers(0, 1 << 62)) << 2 | int(rng.integers(0, 4))
        S = (hi << 64) | (hi ^ _rotl(value, hi >> 58))
        after, _ = R.pcg_raw(S, inc, 2 * MAX_ROUNDS + 2)
        cost, val = R.attempts(np.concatenate([np.array([value], dtype=np.uint64), after]), tab)
        if (cost[0] < 7) if kind == "tail" else (cost[0] != 2 or np.isnan(val[0])):
            continue
        s0 = R.pcg_advance(S, inc, (1 << 128) - (p + 1))
        raw, _ = R.pcg_raw(s0, inc, p + 1 + len(after))
        assert int(raw[p]) == value
        cost, val = R.attempts(raw, tab)
        if R.attempt_starts(cost, val)[p]:
            return s0
    raise AssertionError(f"no state plants a live {kind} at draw {p}")


# ---- host plan: what the device must produce, step by step -------------------------------------------------------
def _decision_ulps(raw, tab, pos):
    """The least distance, in ulp of the threshold side, of the slow-path and tail-round decisions at the attempts
    starting at pos."""
    wi, fi, r = tab["wi"], tab["fi"], tab["r"]
    inv_r = 1.0 / r
    worst = math.inf
    for p in pos:
        w = int(raw[p])
        i, rabs = w & 0xFF, (w >> 9) & R.RABS_MASK
        if i == 0:
            q = p + 1
            while True:
                xx = -inv_r * math.log1p(-R._u(raw[q]))
                yy = -math.log1p(-R._u(raw[q + 1]))
                lhs, rhs = yy + yy, xx * xx
                worst = min(worst, abs(lhs - rhs) / np.spacing(rhs))
                q += 2
                if lhs > rhs:
                    break
        else:
            x = float(rabs) * wi[i]
            lhs, rhs = (fi[i - 1] - fi[i]) * R._u(raw[p + 1]) + fi[i], math.exp(-0.5 * x * x)
            worst = min(worst, abs(lhs - rhs) / np.spacing(rhs))
    return worst


def _census(trace, raw, cost, val, starts, used, plant):
    """The scheme's events in one step: windows, capped windows, list cuts, uncapped short windows, restarts past the
    previous window's W; consumed slow / tail attempts straddling a chunk boundary or the window's end; tail rounds."""
    c = {"shape": (trace[0]["W"], trace[0]["T"], trace[0]["C"]), "windows": len(trace),
         "capped": sum(t["W"] == R.WIN_MAX for t in trace), "cuts": sum(t["cut"] for t in trace),
         "short_uncapped": sum(t["W"] < R.WIN_MAX and t["normals"] < t["rem"] for t in trace),
         "restart_past_W": sum(b["start"] > a["start"] + a["W"] for a, b in zip(trace, trace[1:])),
         "slow_chunk_straddle": 0, "tail_chunk_straddle": 0, "slow_end_straddle": 0, "tail_end_straddle": 0,
         "max_tail_rounds": 0}
    idx0 = (raw & np.uint64(0xFF)) == 0
    for t in trace:
        s, C, weff = t["start"], t["C"], t["weff"]
        for p in np.flatnonzero(starts[s:s + weff] & (cost[s:s + weff] != 1)) + s:
            if p >= used:
                break
            kind = "tail" if idx0[p] else "slow"
            last = p + int(cost[p]) - 1
            if last >= s + weff:
                c[f"{kind}_end_straddle"] += 1
            elif (last - s) // C != (p - s) // C:
                c[f"{kind}_chunk_straddle"] += 1
            if kind == "tail":
                c["max_tail_rounds"] = max(c["max_tail_rounds"], (int(cost[p]) - 1) // 2)
    if plant:
        p = plant[1]
        c["planted_live"] = int(bool(starts[p]))
        c["planted_consumed"] = int(bool(starts[p]) and p < used)
        c["planted_cost"] = int(cost[p])
    return c


@dataclass
class Step:
    state: int                 # the PCG64 state before the step
    normals: np.ndarray        # the sequential oracle's m normals
    tail: np.ndarray           # which of them are idx-0 tail values
    used: int                  # draws consumed
    census: dict


@functools.lru_cache(maxsize=None)
def _plan(name):
    """The case's steps on the host: start state, the sequential normals and draws consumed, the window scheme's
    trace; fails if a guard does not hold."""
    case = CASES[name]
    tab = _table(case.table)
    m = 6 * case.P
    s, inc = R.pcg_state(case.seed)
    if case.plant:
        s = _plant(tab, inc, case.plant[1], case.plant[0], np.random.default_rng(case.seed))
    steps = []
    for k in range(case.steps):
        n = 2 * m + 4096
        while True:
            raw, _ = R.pcg_raw(s, inc, n)
            trace = []
            try:
                got, used_w = R.window_normals(raw, m, tab, trace=trace)
            except ValueError:
                assert n < 64 * m + (1 << 20), f"{name} step {k + 1}: the stream outruns every bound"
                n *= 2
                continue
            assert len(trace) <= MAX_WINDOWS, f"{name} step {k + 1}: {len(trace)} windows"
            classified = max(t["start"] + t["W"] for t in trace)
            if n >= classified + 2 * MAX_ROUNDS + 2:
                break
            n = classified + 2 * MAX_ROUNDS + 2
        cost, val = R.attempts(raw, tab)
        # every position the device classifies: its attempt ends inside raw, and a tail there runs <= 32 rounds
        for t in trace:
            c = cost[t["start"]:t["start"] + t["W"]]
            i0 = (raw[t["start"]:t["start"] + t["W"]] & np.uint64(0xFF)) == 0
            assert (c > 0).all() and (c[i0] <= 1 + 2 * MAX_ROUNDS).all(), f"{name} step {k + 1}: a tail of > 32 rounds"
        want, used = R.normals_from_raw(raw, m, tab)
        assert used == used_w and np.array_equal(got.view(np.uint64), want.view(np.uint64)), \
            f"{name} step {k + 1}: the window scheme differs from the sequential stream"
        if case.table == "real":      # numpy itself on the same state
            g = np.random.Generator(np.random.PCG64())
            g.bit_generator.state = {"bit_generator": "PCG64", "state": {"state": s, "inc": inc},
                                     "has_uint32": 0, "uinteger": 0}
            assert np.array_equal(g.standard_normal(m).view(np.uint64), want.view(np.uint64)), f"{name} step {k + 1}"
            assert int(g.bit_generator.state["state"]["state"]) == R.pcg_advance(s, inc, used), f"{name} step {k + 1}"
        starts = R.attempt_starts(cost, val)
        pos = np.flatnonzero(starts[:used] & ~np.isnan(val[:used]))
        assert len(pos) == m
        consumed = np.flatnonzero(starts[:used] & (cost[:used] != 1))
        ulps = _decision_ulps(raw, tab, consumed)
        assert ulps > MIN_ULPS, f"{name} step {k + 1}: a consumed decision {ulps} ulp from its threshold"
        census = _census(trace, raw, cost, val, starts, used, case.plant if k == 0 else ())
        census["min_decision_ulps"] = ulps
        steps.append(Step(s, want, ((raw[pos] & np.uint64(0xFF)) == 0) & (cost[pos] > 1), used, census))
        s = R.pcg_advance(s, inc, used)
    return tab, inc, steps, s


# ---- host checks (no GPU) ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_case_reaches_its_event_and_the_window_scheme_equals_the_sequential_stream(name):
    """The plan asserts, every step, that the window scheme equals the sequential stream (normals and draws consumed)
    and, on numpy's tables, numpy's Generator; here the first step must reach the event the case is named for."""
    case = CASES[name]
    _, _, steps, _ = _plan(name)
    census = steps[0].census
    print(f"census {name} (m = {6 * case.P}): {census}; windows per step {[st.census['windows'] for st in steps]}")
    assert census["shape"] == SHAPES[case.P]
    assert census[case.event] >= case.at_least, (case.event, census)
    if case.plant:
        kind, p = case.plant
        assert census["planted_live"]
        assert census["planted_cost"] >= 7 if kind == "tail" else census["planted_cost"] == 2


def test_the_cases_reach_every_rare_path():
    first = [_plan(name)[2][0].census for name in CASES]
    total = {k: sum(c[k] for c in first) for k in ("cuts", "short_uncapped", "restart_past_W", "tail_end_straddle",
                                                    "slow_end_straddle", "tail_chunk_straddle", "slow_chunk_straddle")}
    print(f"first steps of all cases: {total}")
    assert all(v > 0 for v in total.values()), total
    # a consumed tail straddling the end of a capped window
    assert any(c["tail_end_straddle"] and c["capped"] for c in first)


def test_kernel_constants_equal_the_restatement():
    src = open(K_MD).read()

    def const(name):
        found = re.findall(rf"\b{name}\s*=\s*(\d+)\b", src)
        assert len(found) == 1, name
        return int(found[0])
    assert const("NZ_WIN") == R.WIN_MAX
    assert const("NZ_MIN_CHUNK") == R.WIN_MIN_CHUNK
    assert const("NZ_LIST") == R.WIN_LIST
    assert const("MD_K1_THREADS") == R.WIN_THREADS       # the block that runs md_refnoise_cta


def test_device_tail_start_is_numpys_r():
    """The device takes the tail start r from wi[255] (layer 255's x at rabs = 2^52); on numpy's tables that is numpy's
    own r, so the stress tables set r the same way."""
    tab = R.tables()
    assert tab["r"] == tab["wi"][255] * 2.0 ** 52


# ---- on the device ---------------------------------------------------------------------------------------------------
def _bare(real_weights, P, state, inc, tab, fr=0.0):
    """An engine with Chignolin's fragments and an empty protein map of P atoms (ef = 0), MD set up on P atoms and the
    reference stream at (state, inc) on the tables tab.  Friction 0: the stream advances, the normals stay out of the
    dynamics."""
    fd = load_fragments("chig")[0]
    eng = Engine(real_weights, 0)
    eng.set_topology(fd.z, fd.batch, n_graphs=len(fd))
    eng.set_protein_map(P, [], [], [], np.zeros(len(fd), np.float32))
    eng.forward_host(np.asarray(fd.pos, dtype=np.float32))
    ef = torch.zeros(3 * P + 1, dtype=torch.float32, device="cuda")
    n = len(fd.z)
    zero = np.zeros(n, np.int32)
    rng = np.random.default_rng(1)
    m = np.array([MASSES[int(a)] for a in rng.choice([1, 6, 7, 8, 16], size=P)])
    eng.md_setup(m, np.arange(n) % P, zero, zero, np.zeros(n, np.float32), FS, KT, fr, 0, ef.data_ptr())
    eng.md_set_state(rng.normal(size=(P, 3)) * 10, rng.normal(size=(P, 3)) * 0.01, 0)
    eng.md_set_noise(1, state, inc, tab)
    return eng, ef


def _check_normals(got, want, tail, what):
    """Bit-identical except idx-0 tail values, within 2 ulp there (the device's log1p)."""
    diff = got.view(np.uint64) != want.view(np.uint64)
    assert not (diff & ~tail).any(), what
    ulps = np.abs(got.view(np.int64) - want.view(np.int64))
    assert (ulps[diff] <= 2).all(), (what, ulps[diff])
    return int(tail.sum()), int(diff.sum()), int(ulps.max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_device_stream_equals_the_sequential_stream(real_weights, name):
    t0 = time.perf_counter()
    case = CASES[name]
    tab, inc, steps, s_last = _plan(name)          # every guard holds before anything is launched
    t_host = time.perf_counter() - t0
    eng, ef = _bare(real_weights, case.P, steps[0].state, inc, tab)
    st = torch.cuda.current_stream().cuda_stream
    after = [s.state for s in steps[1:]] + [s_last]
    tails = differ = worst = 0
    for k, step in enumerate(steps):
        eng.md_run(1, st)
        assert eng.md_get_noise_state() == after[k], f"{name} step {k + 1}: state"
        xi, eta = eng.md_get_noise()
        t, d, u = _check_normals(np.stack([xi, eta]).reshape(-1), step.normals, step.tail, f"{name} step {k + 1}")
        tails, differ, worst = tails + t, differ + d, max(worst, u)
    print(f"measured {name}: {len(steps)} steps, census of step 1 {steps[0].census}; {tails} tail values, "
          f"{differ} differ (max {worst} ulp); host {t_host:.2f} s, total {time.perf_counter() - t0:.2f} s")
