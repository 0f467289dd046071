"""The reference's Langevin noise: numpy's ``default_rng(seed)`` stream (PCG64 + numpy's 256-layer ziggurat).

The reference feeds ASE's ``Langevin.step`` from ``RNGPool(seed)`` (``src/utils/utils.py:28-49``), which pre-draws
``(N, 3)`` arrays with ``np.random.default_rng(seed).standard_normal``; each step consumes two of them, xi then eta.
The device MD step can generate that stream itself (``csrc/k_md.cuh`` ``md_refnoise_cta``); this module gives it what
it needs and restates it on the host:

* :func:`tables` recovers numpy's own ziggurat tables ``wi`` / ``ki`` / ``fi`` and the tail constant ``r`` through the
  public bit-generator API, once per process.  The tables are not recomputed from the ziggurat's defining constants:
  numpy's ``wi`` differs from any recomputation by about 1e-14 relative, which moves the last bits of almost every
  normal.  A bit generator's state is set so that its next outputs are chosen raw values (PCG64: the state whose
  XSL-RR output is the value, stepped back by one LCG step; SFC64: a state whose first two outputs are chosen), and
  ``Generator.standard_normal`` is asked what it does with them:

  - ``rabs = 1`` returns ``wi[idx]`` itself (with ``u = 0`` where that takes the slow path);
  - ``ki[idx]`` is the least ``rabs`` for which the call consumes more than one draw (bisection);
  - ``fi[idx]`` enters only the slow-path test ``(fi[idx-1] - fi[idx]) u + fi[idx] < exp(-x^2 / 2)``: the ``u`` at
    which that test flips is found by bisection for several ``x`` per layer, and ``fi`` is the value next to
    ``exp(-x_idx^2 / 2)`` that reproduces every flip;
  - ``r`` is the idx-0 tail's value at ``u = 0``.

* :func:`attempts` / :func:`normals_from_raw` restate numpy's ``random_standard_normal`` on a given raw 64-bit
  stream (the sequential algorithm), :func:`window_normals` restates the device kernel's parallel window scheme on the
  same stream, and :func:`pcg_advance` is Brown's jump-ahead as the device does it.

Generator streams are not promised stable across numpy releases; the golden fixture records the numpy version it
was made with.
"""
from __future__ import annotations

import functools
import math

import numpy as np

PCG_MULT = 0x2360ED051FC65DA44385DF649FCCF645
M128 = (1 << 128) - 1
M64 = (1 << 64) - 1
RABS_MASK = (1 << 52) - 1
TWO53_INV = 1.0 / 9007199254740992.0

# the device kernel's window scheme (k_md.cuh md_refnoise_cta); window_normals restates it with the same constants
WIN_THREADS = 1024
WIN_MAX = 32768          # draws per window at most
WIN_MIN_CHUNK = 4        # draws per thread at least
WIN_LIST = 1024          # non-fast positions one window can hold; a window with more stops at the first it cannot hold


def window_size(remaining: int) -> int:
    """Draws in the next window for ``remaining`` normals still to make (the result does not depend on it)."""
    return min(WIN_MAX, remaining + (remaining * 3 + 99) // 100 + 64)


# ---- PCG64 (numpy's PCG64: 128-bit LCG, step then XSL-RR output) -------------------------------------------
def pcg_state(seed: int):
    """(state, inc) of ``np.random.PCG64(seed)``."""
    st = np.random.PCG64(seed).state["state"]
    return int(st["state"]), int(st["inc"])


def pcg_output(s: int) -> int:
    hi, lo = s >> 64, s & M64
    rot = hi >> 58
    v = hi ^ lo
    return ((v >> rot) | (v << ((64 - rot) & 63))) & M64


def pcg_advance(s: int, inc: int, k: int) -> int:
    """The state k steps on (Brown, "Random number generation with arbitrary strides", 1994), as the device does it."""
    acc_mult, acc_plus, cur_mult, cur_plus = 1, 0, PCG_MULT, inc
    k &= M128
    while k:
        if k & 1:
            acc_mult = (acc_mult * cur_mult) & M128
            acc_plus = (acc_plus * cur_mult + cur_plus) & M128
        cur_plus = ((cur_mult + 1) * cur_plus) & M128
        cur_mult = (cur_mult * cur_mult) & M128
        k >>= 1
    return (acc_mult * s + acc_plus) & M128


def pcg_raw(s: int, inc: int, n: int):
    """n raw draws from state s: (uint64 array, state after them)."""
    bg = np.random.PCG64()
    bg.state = {"bit_generator": "PCG64", "state": {"state": s, "inc": inc}, "has_uint32": 0, "uinteger": 0}
    raw = bg.random_raw(n)
    return np.asarray(raw, dtype=np.uint64), int(bg.state["state"]["state"])


# ---- table recovery -----------------------------------------------------------------------------------------
class _Forcer:
    """Generators whose next raw outputs can be chosen: one through PCG64, two through SFC64."""

    def __init__(self):
        self.pcg = np.random.PCG64(0)
        self.g_pcg = np.random.Generator(self.pcg)
        self.inc = int(self.pcg.state["state"]["inc"])
        self.minv = pow(PCG_MULT, -1, 1 << 128)
        self.sfc = np.random.SFC64(0)
        self.g_sfc = np.random.Generator(self.sfc)
        self.inv9 = pow(9, -1, 1 << 64)

    def pcg_normal(self, raw: int):
        """(standard_normal() when the next draw is ``raw``, whether it consumed exactly that one draw)."""
        s1 = raw                                   # hi = 0: rotation 0, output hi ^ lo = raw
        self.pcg.state = {"bit_generator": "PCG64", "state": {"state": ((s1 - self.inc) * self.minv) & M128, "inc": self.inc},
                          "has_uint32": 0, "uinteger": 0}
        x = self.g_pcg.standard_normal()
        return x, int(self.pcg.state["state"]["state"]) == s1

    def sfc_normal(self, r1: int, r2: int):
        """(standard_normal() when the next two draws are r1, r2, draws consumed if at most 2 else 3)."""
        # SFC64 output = a + b + counter; with (a, b, c, counter) = (r1, 0, c, 0) the outputs are r1, then 9 c + 1
        self.sfc.state = {"bit_generator": "SFC64", "state": {"state": np.array([r1, 0, ((r2 - 1) * self.inv9) & M64, 0], dtype=np.uint64)},
                          "has_uint32": 0, "uinteger": 0}
        x = self.g_sfc.standard_normal()
        return x, min(int(self.sfc.state["state"]["state"][3]), 3)


def _slow_accept(fi_prev, fi_i, x, um):
    u = um * TWO53_INV
    return (fi_prev - fi_i) * u + fi_i < math.exp(-0.5 * x * x)


def _neighbours(v: float, n: int):
    """v and the n doubles on either side of it."""
    down, up = [v], [v]
    for _ in range(n):
        down.append(float(np.nextafter(down[-1], -np.inf)))
        up.append(float(np.nextafter(up[-1], np.inf)))
    return down[::-1] + up[1:]


@functools.lru_cache(maxsize=1)
def tables():
    """numpy's ziggurat tables as the device takes them: dict ``wi`` (float64[256]), ``ki`` (uint64[256]), ``fi``
    (float64[256]), ``r`` (the tail start), recovered from this process's numpy (see the module docstring)."""
    f = _Forcer()
    wi = np.empty(256)
    ki = np.zeros(256, dtype=np.uint64)
    for i in range(256):
        wi[i], used = f.sfc_normal(i | (1 << 9), 0)     # layer 1 has ki = 0: its slow path accepts x = wi at u = 0
        assert used <= 2, "numpy's standard_normal no longer returns x = wi[idx] for rabs = 1"
        lo, hi = 0, 1 << 52
        while lo < hi:
            mid = (lo + hi) // 2
            if f.pcg_normal(i | (mid << 9))[1]:
                lo = mid + 1
            else:
                hi = mid
        ki[i] = lo
    # the tail's value at u = 0 is r itself (xx = 0); the second tail draw only has to be non-zero
    r = abs(f.sfc_normal(0 | (int(ki[0]) << 9), 0)[0])
    # fi: the u at which the slow-path test flips, for five x per layer, must be numpy's
    probes = {}
    for i in range(1, 256):
        pts = []
        for rabs in np.linspace(int(ki[i]), RABS_MASK, 5).astype(np.int64):
            rabs = int(rabs)
            acc0 = f.sfc_normal(i | (rabs << 9), 0)[1] == 2
            lo, hi = 0, 1 << 53
            while lo < hi:
                mid = (lo + hi) // 2
                if (f.sfc_normal(i | (rabs << 9), mid << 11)[1] == 2) == acc0:
                    lo = mid + 1
                else:
                    hi = mid
            pts.append((rabs * wi[i], acc0, lo))
        probes[i] = pts

    def consistent(fp, fc, i):
        for x, acc0, b in probes[i]:
            if _slow_accept(fp, fc, x, 0) != acc0:
                return False
            if b > 0 and _slow_accept(fp, fc, x, b - 1) != acc0:
                return False
            if b < (1 << 53) and _slow_accept(fp, fc, x, b) == acc0:
                return False
        return True

    fi = np.empty(256)
    fi[0] = 1.0
    cands = [1.0]
    for i in range(1, 256):
        x_i = float(wi[i]) * 2.0 ** 52
        guess = math.exp(-0.5 * x_i * x_i)
        nxt = []
        for fp in cands:
            nxt += [(fp, fc) for fc in _neighbours(guess, 48) if consistent(fp, fc, i)]
        if not nxt:
            raise RuntimeError(f"no ziggurat fi[{i}] reproduces numpy's slow-path decisions")
        prev = sorted({fp for fp, _ in nxt})
        assert len(prev) == 1, f"fi[{i - 1}] is ambiguous"
        fi[i - 1] = prev[0] if i > 1 else fi[0]
        cands = sorted({fc for _, fc in nxt}, key=lambda v: abs(v - guess))
    fi[255] = cands[0]
    return {"wi": wi, "ki": ki, "fi": fi, "r": float(r)}


# ---- numpy's random_standard_normal on a given raw stream --------------------------------------------------
def _u(raw) -> float:
    return (int(raw) >> 11) * TWO53_INV


def attempts(raw, tab=None):
    """Every position of the raw stream taken as the start of one ziggurat attempt: ``(cost, value)`` arrays, cost the
    draws the attempt consumes (1 fast, 2 slow, 1 + 2k for a k-round idx-0 tail) and value its normal (NaN when the
    slow path rejects and the generator starts over).  Positions whose attempt runs past the end of ``raw`` get cost 0."""
    tab = tables() if tab is None else tab
    wi, ki, fi, r = tab["wi"], tab["ki"], tab["fi"], tab["r"]
    raw = np.asarray(raw, dtype=np.uint64)
    idx = (raw & np.uint64(0xFF)).astype(np.int64)
    neg = ((raw >> np.uint64(8)) & np.uint64(1)).astype(bool)
    rabs = (raw >> np.uint64(9)) & np.uint64(RABS_MASK)
    x = rabs.astype(np.float64) * wi[idx]
    x = np.where(neg, -x, x)
    fast = rabs < ki[idx]
    cost = np.ones(len(raw), dtype=np.int64)
    val = x.copy()
    inv_r = 1.0 / r
    for p in np.flatnonzero(~fast):
        i = int(idx[p])
        if i == 0:
            k, q = 0, p + 1
            while True:
                if q + 1 >= len(raw):
                    cost[p], val[p] = 0, np.nan
                    break
                xx = -inv_r * math.log1p(-_u(raw[q]))
                yy = -math.log1p(-_u(raw[q + 1]))
                k, q = k + 1, q + 2
                if yy + yy > xx * xx:
                    cost[p] = 1 + 2 * k
                    val[p] = -(r + xx) if (int(rabs[p]) >> 8) & 1 else r + xx
                    break
        elif p + 1 >= len(raw):
            cost[p], val[p] = 0, np.nan
        else:
            cost[p] = 2
            xp = float(x[p])
            if not (fi[i - 1] - fi[i]) * _u(raw[p + 1]) + fi[i] < math.exp(-0.5 * xp * xp):
                val[p] = np.nan
    return cost, val


def attempt_starts(cost, val):
    """Positions where the sequential generator starts an attempt: the chain a0 = 0, a(j+1) = a(j) + cost(a(j)),
    which leaves the "+1" path only at non-fast positions.  Returns a boolean mask."""
    live = np.ones(len(cost), dtype=bool)
    cur = 0
    for p in np.flatnonzero((cost != 1) | np.isnan(val)):
        if p < cur:
            continue
        if cost[p] == 0:
            live[p:] = False
            break
        cur = int(p + cost[p])
        live[p + 1:cur] = False
    return live


def normals_from_raw(raw, n: int, tab=None):
    """numpy's ``standard_normal(n)`` on the raw stream, sequentially: (normals, draws consumed)."""
    cost, val = attempts(raw, tab)
    pos = np.flatnonzero(attempt_starts(cost, val) & ~np.isnan(val))
    if len(pos) < n:
        raise ValueError("raw stream too short")
    last = int(pos[n - 1])
    return val[pos[:n]], last + int(cost[last])


def window_normals(raw, n: int, tab=None, list_cap: int = WIN_LIST, trace: list | None = None):
    """The device kernel's scheme (k_md.cuh ``md_refnoise_cta``) on the same stream: windows of ``window_size`` draws,
    each split into contiguous per-thread chunks that are classified independently; the non-fast positions of a window,
    in order, are walked (in runs between anchors on the device) to mark the draws consumed inside other attempts; a
    prefix count over the surviving attempts with a value numbers the normals.  A window holding more than ``list_cap``
    non-fast positions stops at the first it cannot hold, and a window that yields too few normals is followed by
    another from where its attempts ended.  Returns (normals, draws consumed) -- equal to :func:`normals_from_raw`.

    ``trace``, when given, gets one dict per window: ``start`` (its first draw in ``raw``), ``W``, ``T``, ``C``,
    ``weff`` (where the window stops, relative to ``start``), ``cut`` (the list overflowed), ``rem`` (normals still
    wanted), ``normals`` (how many of them it yielded) and ``end`` (the draw the next window or the step starts from)."""
    cost, val = attempts(raw, tab)
    out, base = [], 0
    while len(out) < n:
        rem = n - len(out)
        W = window_size(rem)
        T = min(WIN_THREADS, -(-W // WIN_MIN_CHUNK))
        C = -(-W // T)
        if base + W > len(raw):
            raise ValueError("raw stream too short")
        c, v = cost[base:base + W], val[base:base + W]
        if (c == 0).any():
            raise ValueError("raw stream too short")
        nonfast = (c != 1) | np.isnan(v)
        # per-thread counts of non-fast positions, exclusive scan, the list truncated at list_cap
        nf = [int(nonfast[t * C:min((t + 1) * C, W)].sum()) for t in range(T)]
        lst = np.flatnonzero(nonfast)
        assert len(lst) == sum(nf)
        weff = W if len(lst) <= list_cap else int(lst[list_cap])
        lst = lst[:list_cap]
        # the walk
        dead = np.zeros(W, dtype=bool)
        cur = 0
        for p in lst:
            if p < cur:
                continue
            cur = int(p + c[p])
            dead[p + 1:min(cur, weff)] = True
        end = max(cur, weff)
        hasval = ~dead & ~np.isnan(v)
        hasval[weff:] = False
        got = 0
        for t in range(T):                    # per-thread counts, exclusive scan, scatter
            for i in range(t * C, min((t + 1) * C, W)):
                if hasval[i]:
                    if got < rem:
                        out.append(v[i])
                        if got == rem - 1:
                            end = i + int(c[i])
                    got += 1
        if trace is not None:
            trace.append({"start": base, "W": W, "T": T, "C": C, "weff": weff, "cut": weff < W, "rem": rem,
                          "normals": min(got, rem), "end": base + end})
        base += end
    return np.array(out), base
