"""The persistent TMA-staged stencil kernels with many tiles per CTA.

``k_stencil_row_tma`` (``xg_stencil2(row_tma)``), ``k_tile_stencil`` (``xg_stencil2(tile_tma)`` along Y and, with
rows = Z and levels = Y, along Z; with an x term ``xg_stencil_pair(tile_tma)``) and ``k_tile_multi``
(``xg_stencil_multi(tile_tma)``) are persistent: a grid of at most 4 CTAs per SM walks nrb x nzq x rbq x ntx virtual
tiles through a ring of shared-memory stages guarded by full / empty mbarriers, and skips the row-block slots past
the last tile row.  On small fields every CTA gets one tile, so the empty-barrier wait, the phase flip and the
skipped slots never run.  Every case here gives each CTA at least 8 tiles at the largest grid a launcher may pick,
and each kernel and dtype has a field whose x extent, rows and levels are all ragged and whose last row block has
skipped slots.  Fields carry NaN, +-0 and +-inf; every output cell is compared with the oracle and every call
asserts the kernel label, so a silent fallback to another kernel fails instead of passing.

The launch knobs (a ring of one stage, one CTA per SM, short row blocks, L2 eviction hints) are read once per
process, so each configuration runs a trimmed copy of the sweep in a child process.
"""

import itertools
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import stencil as oracle

DEV = "cuda:0"
NAN = float("nan")

# ---------------------------------------------------------------------------------------------- launch arithmetic
SMS = 132  # H100 SXM (XG_SMS, xg_common.cuh)
MAX_CTAS = 4  # the most CTAs per SM any of the three launchers picks (k_tile_multi without an x op)
MIN_TILES_PER_CTA = 8
U = 4  # levels per tile
GEO = {np.dtype(np.float32): (224, 4), np.dtype(np.float64): (240, 2)}  # (TXE cells, TY rows) per tile


def schedule(dtype, n, rows, levels, rb=128):
    """The virtual tiles of one launch, computed as the launchers compute them: ``launch_row_tma``
    (xg_stencil2.cu, ``ntx`` .. ``a.ntiles``), ``xg_tile_stencil`` (xg_stencil_tile.cu, ``ntx`` .. ``a.ntiles``) and
    ``xg_multi_tile`` (xg_stencil_multi_tma.cu, ``ntx`` .. ``a.ntiles``); ``rb`` is ``XG_*_RB``.  ``rows`` is the
    tile-row extent (the row kernel's P, the tile kernel's output rows Po, the multi kernel's P) and ``levels`` the
    level extent (Zn / L)."""
    txe, ty = GEO[np.dtype(dtype)]

    def cdiv(a, b):
        return -(-a // b)

    ntx = cdiv(n, txe)
    npq = cdiv(rows, ty)
    rbq_target = cdiv(rb if rb > 0 else 128, ty)
    nrb = cdiv(npq, rbq_target)
    rbq = cdiv(npq, nrb)
    nzq = cdiv(levels, U)
    return {"ntiles": nrb * nzq * rbq * ntx, "npq": npq, "nrb": nrb, "rbq": rbq, "nzq": nzq, "ntx": ntx,
            "skipped": nrb * rbq - npq, "ragged": (n % txe != 0, rows % ty != 0, levels % U != 0)}


def test_schedule_mirror_worked_examples():
    """Hand-computed schedules of the sweep's fields."""
    s = schedule(np.float32, 1124, 266, 45)
    assert (s["ntiles"], s["skipped"], s["nrb"], s["rbq"], s["npq"]) == (4968, 2, 3, 23, 67)
    s = schedule(np.float64, 1124, 266, 45)
    assert (s["ntiles"], s["skipped"]) == (8100, 2)
    s = schedule(np.float32, 1124, 129, 100)
    assert (s["ntiles"], s["skipped"]) == (5100, 1)
    assert schedule(np.float64, 1124, 129, 100)["skipped"] == 1
    s = schedule(np.float64, 1124, 137, 101)
    assert (s["ntiles"], s["skipped"]) == (9100, 1)
    assert schedule(np.float32, 1124, 137, 101, rb=12)["skipped"] == 1
    assert schedule(np.float64, 1124, 136, 101)["skipped"] == 0
    s = schedule(np.float32, 1124, 264, 45)
    assert (s["ntiles"], s["skipped"]) == (4752, 0)  # nrb x rbq == npq: the last virtual tile is a real one
    s = schedule(np.float32, 1124, 265, 45, rb=12)
    assert (s["nrb"], s["rbq"], s["skipped"]) == (23, 3, 2)
    assert schedule(np.float32, 1124, 265, 45)["ragged"] == (True, True, True)


# ---------------------------------------------------------------------------------------------- fields and checks
FIELD = (45, 265, 1124)  # X, Y and pair / multi: fp32 4968 tiles (2 skipped slots), fp64 8100 (2 skipped)
FIELD_Z = (137, 101, 1124)  # along Z (rows = Z, levels = Y): fp32 5616 tiles, fp64 9100, 1 skipped slot each
# (also with XG_TILE_RB=12); n_out = n - 1 leaves no slot skipped, so there the last virtual tile is a real one
BCS = [("periodic", 0.0), ("fill", 0.0), ("fill", 1.5), ("fill", NAN), ("extend", 0.0), ("extrapolate", 0.0)]
BCS3 = [b for b in BCS if b[0] != "extrapolate"]  # the pair and multi kernels take periodic / fill / extend
_cache = {}


def _field(shape, dtype, seed):
    """N(0, 1) with 0.4 % NaN, 0.2 % +inf, 0.2 % -inf, 0.4 % +0 and 0.4 % -0 (host array, device copy)."""
    key = ("f", shape, np.dtype(dtype).str, seed)
    if key not in _cache:
        rng = np.random.default_rng(seed)
        a = rng.standard_normal(shape).astype(dtype)
        r = rng.random(shape)
        for lo, hi, v in ((0.0, 0.004, np.nan), (0.004, 0.006, np.inf), (0.006, 0.008, -np.inf), (0.008, 0.012, 0.0),
                          (0.012, 0.016, -0.0)):
            a[(r >= lo) & (r < hi)] = v
        _cache[key] = (a, torch.from_numpy(a).to(DEV))
    return _cache[key]


def _metric(shape, dtype):
    """A positive metric of the given (broadcastable) shape, or (None, None) for ``shape=None``."""
    if shape is None:
        return None, None
    key = ("m", tuple(shape), np.dtype(dtype).str)
    if key not in _cache:
        m = (0.5 + np.random.default_rng(list(shape)).random(shape)).astype(dtype)
        _cache[key] = (m, torch.from_numpy(m).to(DEV))
    return _cache[key]


def _poisoned(shape, dtype):
    """An output buffer whose every cell holds a value no result here can take: a cell a kernel skips fails."""
    return torch.full(tuple(shape), 1.2345e30, dtype=torch.float32 if dtype == np.float32 else torch.float64, device=DEV)


def _expect(label, got, want, sched, ctx):
    from xgcm_b200 import _capi

    seen = _capi.last_launch()
    assert seen == label, f"{ctx}: served by {seen}"
    assert sched["ntiles"] >= MIN_TILES_PER_CTA * MAX_CTAS * SMS, f"{ctx}: {sched}"
    got = got.cpu().numpy()
    assert got.shape == want.shape, ctx
    if not np.array_equal(got, want, equal_nan=True):  # the cheap test first; the report on a mismatch
        np.testing.assert_array_equal(got, want, err_msg=ctx)


def _oracle(fn, *args):
    with np.errstate(all="ignore"):  # inf - inf, inf * 0 ...: NaN on both sides
        return fn(*args)


def _halo_want(op, a, axis, lo, hi, pre, post, hl, hh):
    """OP(concat(halo_lo, A x pre, halo_hi)) / post: explicit halo planes replace the boundary rule."""
    ap = a if pre is None else a * pre
    parts = ([np.expand_dims(hl, axis)] if lo else []) + [ap] + ([np.expand_dims(hh, axis)] if hi else [])
    padded = np.concatenate(parts, axis=axis)
    return (np.moveaxis(oracle.KERNELS[op](np.moveaxis(padded, axis, -1)), -1, axis) / post).astype(a.dtype)


# ---------------------------------------------------------------------------------------------- the cases
# Each list starts with a case whose x, rows and levels are all ragged and whose last row block skips slots, so
# every trimmed copy (cases[::stride]) keeps one.  The parameters not swept in full come from a seeded generator.
def _row_cases():
    """derivative('X')-like: post = dx(Y, X) (rows = Y, levels = Z) or dx(X) (one row, levels = Z x Y)."""
    rng = np.random.default_rng(100)
    pres = ["yx", "none", "full", "x", "row", "level"]
    cases = []
    for post in ("yx", "x"):
        for pre in pres:
            if post == "x" and pre == "yx":
                continue  # levels = Z x Y: a (Y, X) pre-metric has no row of its own (row_zb / row_vec take it)
            for op, lo in itertools.product(("diff", "interp"), (1, 0)):
                cases.append({"pre": pre, "post": post, "op": op, "lo": lo, "bc": BCS[rng.integers(len(BCS))]})
    return cases


def _tile_cases(swap):
    """Along Y (rows = Y', levels = Z) or, with ``swap``, along Z (rows = Z', levels = Y): every shift (n_out = n - 1,
    n, n + 1), every metric layout the tile kernel stages, a few explicit halo planes."""
    rng = np.random.default_rng(200 + swap)
    shifts = [(1, 0), (0, 1), (1, 1), (0, 0)]
    ops_ = ["diff", "interp", "diff", "interp", "max", "min"]
    cases = []
    if swap:  # the divisor must be one scalar per row (dz(Z)); pre: none, per row, or the full field
        for (lo, hi), pre in itertools.product(shifts, ("level", "none", "full")):
            cases.append({"lo": lo, "hi": hi, "pre": pre, "post": "level"})
    else:
        pres = ["yx", "none", "full", "level", "x", "row"]
        k = 0
        for (lo, hi), post in itertools.product(shifts, ("yx", "x", "row", "level")):
            for _ in range(2):
                cases.append({"lo": lo, "hi": hi, "pre": pres[k % len(pres)], "post": post})
                k += 1
            if post == "yx":
                cases.append({"lo": lo, "hi": hi, "pre": "yx", "post": "full"})
    for c in cases:
        c["op"] = ops_[rng.integers(len(ops_))]
        c["bc"] = BCS[rng.integers(len(BCS))]
    for lo, hi in ((1, 0), (0, 1), (1, 1)):
        cases.append({"lo": lo, "hi": hi, "pre": "level" if swap else "yx", "post": "level" if swap else "yx",
                      "op": "interp" if hi else "diff", "bc": ("fill", 2.5), "halo": True})
    return cases


PAIR_METRICS = [("yx", "yx", "yx"), ("full", "yx", "yx"), ("level", "full", "yx"), ("none", "yx", "none"),
                ("yx", "none", "yx"), ("x", "row", "yx"), ("row", "x", "x"), ("none", "none", "yx"),
                ("yx", "yx", "level"), ("yx", "yx", "row"), ("full", "full", "full"), ("yx", "full", "full")]


def _pair_cases():
    """(OPa(u x pre_a) along X +|- OPb(v x pre_b) along Y) / post: every subtract form and metric combo."""
    rng = np.random.default_rng(300)
    ops_ = [("diff", "diff"), ("interp", "diff"), ("diff", "interp"), ("interp", "interp")]
    cases = []
    for (pre_a, pre_b, post), sub in itertools.product(PAIR_METRICS, (0, 1, 2)):
        cases.append({"pre_a": pre_a, "pre_b": pre_b, "post": post, "sub": sub, "ops": ops_[rng.integers(4)],
                      "lo": (int(rng.integers(2)), int(rng.integers(2))),
                      "bcs": (BCS3[rng.integers(len(BCS3))], BCS3[rng.integers(len(BCS3))])})
    return cases


def _multi_cases():
    """interp / diff / min / max over {x, y, z}, {x, y}, {x, z} and {y, z} (no x op: one stage, 4 CTAs per SM)."""
    rng = np.random.default_rng(400)
    cases = []
    for axes, op in itertools.product([(2, 1, 0), (2, 1), (2, 0), (1, 0)], ("interp", "diff", "min", "max")):
        cases.append({"axes": axes, "op": op, "los": [int(rng.integers(2)) for _ in axes],
                      "bcs": [BCS3[rng.integers(len(BCS3))] for _ in axes]})
    return cases


# ---------------------------------------------------------------------------------------------- the runners
def _shape_of(kind, shape):
    Z, Y, X = shape
    return {"none": None, "full": (Z, Y, X), "yx": (1, Y, X), "x": (1, 1, X), "row": (1, Y, 1), "level": (Z, 1, 1),
            "zrow": (Z, Y, 1)}[kind]


def _run_row(dtype, c, rb):
    from xgcm_b200 import ops

    Z, Y, X = FIELD
    a, ta = _field(FIELD, dtype, 1)
    pre, tpre = _metric(_shape_of("zrow" if c["pre"] == "row" else c["pre"], FIELD), dtype)
    post, tpost = _metric(_shape_of(c["post"], FIELD), dtype)
    lo, hi = c["lo"], 1 - c["lo"]
    bc, fill = c["bc"]
    sched = schedule(dtype, X, Y, Z, rb) if c["post"] == "yx" else schedule(dtype, X, 1, Z * Y, rb)
    out = _poisoned(FIELD, dtype)
    ops.stencil2(ta, 2, c["op"], lo, hi, bc, fill, pre=tpre, post=tpost, out=out)
    want = _oracle(oracle.stencil2, c["op"], a, 2, lo, hi, bc, fill, pre, post)
    _expect("xg_stencil2(row_tma)", out, want, sched, f"row_tma {np.dtype(dtype)} {c}")
    return sched


def _run_tile(dtype, c, rb, swap):
    from xgcm_b200 import ops

    shape = FIELD_Z if swap else FIELD
    axis = 0 if swap else 1
    a, ta = _field(shape, dtype, 2)
    lo, hi = c["lo"], c["hi"]
    n_out = shape[axis] + lo + hi - 1
    oshape = list(shape)
    oshape[axis] = n_out
    pre, tpre = _metric(_shape_of(c["pre"], shape), dtype)
    post, tpost = _metric(_shape_of(c["post"], oshape), dtype)
    bc, fill = c["bc"]
    rows, levels = (n_out, shape[1]) if swap else (n_out, shape[0])
    sched = schedule(dtype, shape[2], rows, levels, rb)
    out = _poisoned(oshape, dtype)
    if c.get("halo"):
        plane = [s for d, s in enumerate(shape) if d != axis]
        hl, thl = _metric(tuple(plane), dtype)
        hh = (hl[::-1] * 1.5).astype(dtype)
        ops.stencil2(ta, axis, c["op"], lo, hi, bc, fill, pre=tpre, post=tpost, halo_lo=thl if lo else None,
                     halo_hi=torch.from_numpy(hh).to(DEV) if hi else None, out=out)
        want = _oracle(_halo_want, c["op"], a, axis, lo, hi, pre, post, hl, hh)
    else:
        ops.stencil2(ta, axis, c["op"], lo, hi, bc, fill, pre=tpre, post=tpost, out=out)
        want = _oracle(oracle.stencil2, c["op"], a, axis, lo, hi, bc if (lo or hi) else None, fill, pre, post)
    _expect("xg_stencil2(tile_tma)", out, want, sched, f"tile_tma({'Z' if swap else 'Y'}) {np.dtype(dtype)} {c}")
    return sched


def _run_pair(dtype, c, rb):
    from xgcm_b200 import ops

    Z, Y, X = FIELD
    a, ta = _field(FIELD, dtype, 3)
    b, tb = _field(FIELD, dtype, 4)
    (pa, tpa), (pb, tpb), (po, tpo) = (_metric(_shape_of(k, FIELD), dtype) for k in (c["pre_a"], c["pre_b"], c["post"]))
    (op_a, op_b), (lo_a, lo_b), ((bc_a, fa), (bc_b, fb)) = c["ops"], c["lo"], c["bcs"]
    sched = schedule(dtype, X, Y, Z, rb)
    got = ops.stencil_pair(ta, tb, (op_a, lo_a, 1 - lo_a, bc_a, fa), (1, op_b, lo_b, 1 - lo_b, bc_b, fb), c["sub"],
                           pre_a=tpa, pre_b=tpb, post=tpo)
    want = _oracle(oracle.stencil_pair, op_a, a, 2, lo_a, 1 - lo_a, bc_a, fa, pa, op_b, b, 1, lo_b, 1 - lo_b, bc_b, fb,
                   pb, c["sub"], po)
    _expect("xg_stencil_pair(tile_tma)", got, want, sched, f"pair {np.dtype(dtype)} {c}")
    return sched


def _run_multi(dtype, c, rb):
    from xgcm_b200 import ops

    Z, Y, X = FIELD
    a, ta = _field(FIELD, dtype, 5)
    specs = [(ax, c["op"], lo, 1 - lo, bc, fill) for ax, lo, (bc, fill) in zip(c["axes"], c["los"], c["bcs"])]
    sched = schedule(dtype, X, Y, Z, rb)
    got = ops.stencil_multi(ta, specs)
    want = a
    for ax, op, lo, hi, bc, fill in specs:
        want = _oracle(oracle.stencil2, op, want, ax, lo, hi, bc, fill)
    _expect("xg_stencil_multi(tile_tma)", got, want, sched, f"multi {np.dtype(dtype)} {specs}")
    return sched


KERNELS = {
    "row_tma": (_row_cases, _run_row),
    "tile_tma(Y)": (lambda: _tile_cases(False), lambda d, c, rb: _run_tile(d, c, rb, False)),
    "tile_tma(Z)": (lambda: _tile_cases(True), lambda d, c, rb: _run_tile(d, c, rb, True)),
    "pair": (_pair_cases, _run_pair),
    "multi": (_multi_cases, _run_multi),
}


def run_sweep(kernel, dtype, stride=1, rb=128, tag="default"):
    """Every ``stride``-th case of one kernel in one dtype; prints the schedules met and returns them."""
    make, run = KERNELS[kernel]
    seen = {}
    for c in make()[::stride]:
        s = run(dtype, c, rb)
        key = (s["ntiles"], s["skipped"], s["ragged"])
        seen[key] = seen.get(key, 0) + 1
    _cache.clear()
    # the sweep reached what it is for: several tiles per CTA everywhere (_expect), skipped slots and ragged tiles in
    # x, rows and levels — in one field at the default row blocks; short row blocks move the skipped slots elsewhere
    if rb == 128:
        assert any(skipped > 0 and all(ragged) for _, skipped, ragged in seen), (kernel, seen)
    else:
        assert any(skipped > 0 for _, skipped, _ in seen) and any(all(r) for _, _, r in seen), (kernel, seen)
    for (ntiles, skipped, ragged), calls in sorted(seen.items()):
        print(f"[tma-schedule] {tag} {kernel} {np.dtype(dtype)}: ntiles={ntiles} "
              f">= {ntiles / (MAX_CTAS * SMS):.1f} tiles per CTA at {MAX_CTAS} x {SMS} CTAs, "
              f"{skipped} skipped slots, ragged x/rows/levels={ragged}, {calls} calls")
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_tma_ring_many_tiles_per_cta(kernel, dtype):
    run_sweep(kernel, dtype)


# ---------------------------------------------------------------------------------------------- launch knobs
KNOBS = {
    "nst1": {"XG_ROW_TMA_NST": "1", "XG_TILE_NST": "1", "XG_MULTI_NST": "1"},  # every tile after the first waits on empty
    "ctas1": {"XG_ROW_TMA_CTAS": "1", "XG_TILE_CTAS": "1", "XG_MULTI_CTAS": "1"},  # more tiles per CTA
    "rb12": {"XG_ROW_TMA_RB": "12", "XG_TILE_RB": "12", "XG_MULTI_RB": "12"},  # many row blocks, many skipped slots
    "hint": {"XG_ROW_TMA_HINT": "1", "XG_TILE_HINT": "1"},  # tensor loads with L2 eviction hints
}


@pytest.mark.gpu
@pytest.mark.parametrize("knob", list(KNOBS))
def test_tma_ring_launch_knobs(knob):
    """A trimmed sweep of every kernel and dtype in a child process started with the knob set."""
    env = dict(os.environ)
    env.update(KNOBS[knob])
    rb = 12 if knob == "rb12" else 128
    tests_dir = os.path.dirname(os.path.abspath(__file__))
    code = (
        "import sys\n"
        f"sys.path[:0] = [{os.path.dirname(tests_dir)!r}, {tests_dir!r}]\n"
        "import numpy as np\n"
        "import test_tma_schedule_gpu as t\n"
        "for k in t.KERNELS:\n"
        "    for dt in (np.float32, np.float64):\n"
        f"        t.run_sweep(k, dt, stride=8, rb={rb}, tag={knob!r})\n"
    )
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, f"{knob}: exit {r.returncode}\n{r.stdout[-4000:]}\n{r.stderr[-8000:]}"
