"""Every compiled kernel instance against the oracle.

The build writes ``kernels.txt`` (``xgcm_b200/_build.py``): one line per ``__global__`` instance linked into the
library, demangled the way the CUDA profiler names kernels.  The GPU sweep below drives the public entry points
(``ops.*`` and their host twins) across dtype, operator, shift, boundary, metric layout, shapes either side of every
vector / TMA / tile threshold, ragged rows and base pointers 1-3 elements (fp32) or 1 element (fp64) off a 16-byte
boundary, checks every result against the oracle and records, under ``torch.profiler``, which kernels ran.  The
last test asserts that every instance in the manifest ran except the ones in ``ALLOWLIST``.

The misaligned views are what a user passes when slicing ``x[t]`` out of a (T, Z, Y, X) field with an odd
Z * Y * X, and what the host pipelines hand the kernels for plane offsets; they take the scalar and non-TMA routes
that an aligned tensor of the same size never takes.
"""

from __future__ import annotations

import itertools
import math
import re
from collections import defaultdict

import numpy as np
import pytest

from oracle import stencil as oracle

DEV = "cuda:0"
NAN = float("nan")

# instances no single-GPU input reaches, with the reason
_COMM = "xg_comm: NCCL halo exchange between two GPUs (test_parallel_gpu.py needs a second device)"
_WIDTHS = (("float", 1), ("float", 4), ("double", 1), ("double", 2))
ALLOWLIST = {
    **{f"k_edge_fix<{t}, {v}, {o}>": _COMM for t, v in _WIDTHS for o in range(4)},
    **{f"k_pack_plane<{t}, {v}>": _COMM for t, v in _WIDTHS},
}


def _key(name: str) -> str:
    """``void (anonymous namespace)::k_x<float, 1>((anonymous namespace)::Args<float>)`` -> ``k_x<float, 1>``."""
    name = name.strip()
    if name.startswith("void "):
        name = name[5:]
    name = re.sub(r"^(?:\w+::)*(?:\(anonymous namespace\)::)?(?:\w+::)*", "", name)
    name = name.replace("(anonymous namespace)::", "")
    depth = 0
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
            if depth == 0:
                return name[: i + 1]
    return name.split("(")[0]


def _manifest():
    from xgcm_b200 import _build

    path = _build.BUILD_DIR / "kernels.txt"
    if not path.exists():
        pytest.fail(f"{path} is missing: build the library with `python -m xgcm_b200._build`")
    return _build.read_manifest(path)


# ---------------------------------------------------------------------------------------------- the manifest (CPU)
def test_manifest_matches_build_and_allowlist():
    """The manifest belongs to the sources as they are, parses, and its per-file counts and allowlisted names agree."""
    from xgcm_b200 import _build

    digest, entries = _manifest()
    assert digest == _build.current_digest(), "kernels.txt is stale: rebuild the library"
    assert (_build.BUILD_DIR / "digest.txt").read_text() == digest
    keys = [_key(n) for _, n in entries]
    assert len(set(keys)) == len(keys), "two instances share a name"
    per_file = defaultdict(int)
    for stem, _ in entries:
        per_file[stem] += 1
    assert dict(per_file) == {
        "xg_comm": 20, "xg_cumscan": 16, "xg_elementwise": 28, "xg_faces": 4, "xg_fold": 2, "xg_stencil2": 96,
        "xg_stencil_multi": 112, "xg_stencil_multi_tma": 56, "xg_stencil_pair": 40, "xg_stencil_tile": 32,
        "xg_vconserv": 2, "xg_vinterp": 4, "xg_vinterp_tma": 6, "xg_wreduce": 16,
    }
    comm = {_key(n) for s, n in entries if s == "xg_comm"}
    assert set(ALLOWLIST) == comm, "the allowlist names exactly the two-GPU instances"
    # only the (K, LAST, MARCH) triples multi_typed can select are compiled (xg_stencil_multi.cu launch_march)
    triples = {tuple(int(v) for v in k.split(", ")[2:5]) for k in keys if k.startswith("k_stencil_multi<")}
    assert triples == {(2, -1, 1), (2, 0, 1), (2, 1, 0), (3, -1, 2), (3, 0, 2), (3, 1, 2), (3, 2, 1)}


def test_key_normalises_profiler_names():
    assert _key("void (anonymous namespace)::k_scan_rows<double, false>((anonymous namespace)::ScanArgs<double>)") \
        == "k_scan_rows<double, false>"
    assert _key("void xgvi::(anonymous namespace)::k_vinterp_shared_tma<float, 2>(CUtensorMap, "
                "xgvi::(anonymous namespace)::InterpArgs<float>)") == "k_vinterp_shared_tma<float, 2>"


# ---------------------------------------------------------------------------------------------- GPU helpers
_LAUNCHED: dict = {}  # sweep test name -> set of kernel keys it launched


class _Capture:
    """Collects the names of the CUDA kernels launched inside the block (torch.profiler, CUDA activities)."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.synchronize()
        self.prof = profile(activities=[ProfilerActivity.CUDA])
        self.prof.__enter__()
        return self

    def __exit__(self, *exc):
        import torch

        torch.cuda.synchronize()
        self.prof.__exit__(*exc)
        if exc[0] is None:
            names = {_key(e.name) for e in self.prof.events() if e.name.startswith("void ")}
            _LAUNCHED.setdefault(self.name, set()).update(names)
        return False


def _tdt(dtype):
    import torch

    return torch.float32 if np.dtype(dtype) == np.float32 else torch.float64


def _offsets(dtype):
    """Element offsets of a view from a 16-byte aligned base: aligned, then every misalignment the dtype allows."""
    return (0, 1, 2, 3) if np.dtype(dtype) == np.float32 else (0, 1)


def _dev(a, off=0):
    """A device copy of ``a`` that starts ``off`` elements past a 16-byte aligned allocation: ``base[k:k+n].view``."""
    import torch

    if a is None:
        return None
    a = np.ascontiguousarray(a)
    base = torch.empty(a.size + off + 1, dtype=_tdt(a.dtype), device=DEV)
    assert base.data_ptr() % 16 == 0
    v = base[off:off + a.size].view(a.shape)
    v.copy_(torch.from_numpy(a))
    assert v.data_ptr() % 16 == off * a.itemsize
    return v


SENTINEL = 1.2345e30  # no result here can take this value
_GUARDED = []  # (allocation, first cell of the view, cells in the view) of every _empty not yet checked


def _empty(shape, dtype, off=0):
    """An output view ``off`` elements past a 16-byte boundary, with a 16-byte guard band on each side; every cell
    holds SENTINEL.  ``_eq`` checks that the guard bands still hold it after the call."""
    import torch

    n = int(np.prod(shape))
    g = 16 // np.dtype(dtype).itemsize
    base = torch.full((g + off + n + g,), SENTINEL, dtype=_tdt(dtype), device=DEV)
    _GUARDED.append((base, g + off, n))
    return base[g + off:g + off + n].view(tuple(shape))


def _check_guards(ctx):
    for base, start, n in _GUARDED:
        assert bool((base[:start] == SENTINEL).all()), f"{ctx}: a store landed before the output view"
        assert bool((base[start + n:] == SENTINEL).all()), f"{ctx}: a store landed past the output view"
    _GUARDED.clear()


def _field(shape, dtype, seed, specials=True):
    """N(0, 1) with NaN, +-inf and +-0 sprinkled in (0.3 % each)."""
    rng = np.random.default_rng(seed)
    a = rng.standard_normal(shape).astype(dtype)
    if specials:
        r = rng.random(shape)
        a[r < 0.003] = np.nan
        a[(r >= 0.003) & (r < 0.006)] = np.inf
        a[(r >= 0.006) & (r < 0.009)] = -np.inf
        a[(r >= 0.009) & (r < 0.012)] = 0.0
        a[(r >= 0.012) & (r < 0.015)] = -0.0
    return a


def _metric(shape, dtype, seed):
    return None if shape is None else (0.5 + np.random.default_rng(seed).random(shape)).astype(dtype)


def _eq(got, want, ctx):
    _check_guards(ctx)
    got = got.cpu().numpy() if hasattr(got, "cpu") else np.asarray(got)
    assert got.shape == want.shape, f"{ctx}: shape {got.shape} != {want.shape}"
    assert got.dtype == want.dtype, f"{ctx}: dtype {got.dtype} != {want.dtype}"
    np.testing.assert_array_equal(got, want, err_msg=ctx)


def _layout(kind, shape):
    """Broadcast shapes of a metric against ``shape``: the layouts the launchers tell apart."""
    nd = len(shape)
    if kind is None:
        return None
    if kind == "full":
        return tuple(shape)
    if kind == "lead1":  # shared between levels: dx(Y, X) of a (Z, Y, X) field
        return (1,) + tuple(shape[1:])
    if kind == "last":  # dx(X)
        return (1,) * (nd - 1) + (shape[-1],)
    if kind == "first":  # dz(Z)
        return (shape[0],) + (1,) * (nd - 1)
    if kind == "nolast":  # one scalar per row
        return tuple(shape[:-1]) + (1,)
    raise ValueError(kind)


METRICS = [(None, None), (None, "lead1"), ("full", "lead1"), ("lead1", "lead1"), ("first", None),
           ("nolast", "last"), ("last", "full"), ("lead1", None), ("first", "first"), (None, "last")]
BCS = [("periodic", 0.0), ("fill", 0.0), ("fill", 1.5), ("fill", NAN), ("extend", 0.0), ("extrapolate", 0.0)]
BCS3 = [b for b in BCS if b[0] != "extrapolate"]
SHIFTS = [(1, 0), (0, 1), (1, 1), (0, 0)]
OPS = ("diff", "interp", "min", "max")
DTYPES = (np.float32, np.float64)


def _stencil_shapes(dtype):
    # x past the TMA threshold (2 * 224 fp32 / 2 * 240 fp64 cells) and a multiple of the vector width; the same
    # ragged; x long enough for row_vec only; short rows; a fourth dim that splits the inner block
    return [(4, 6, 520), (4, 6, 517), (3, 5, 136), (3, 5, 7), (2, 3, 4, 136), (70, 33)]


def _oracle(fn, *args, **kw):
    with np.errstate(all="ignore"):
        return fn(*args, **kw)


def _halo_want(op, a, axis, lo, hi, pre, post, hl, hh):
    """OP(concat(halo_lo, A x pre, halo_hi)) / post: explicit halo planes replace the boundary rule."""
    ap = a if pre is None else a * pre
    parts = ([np.expand_dims(hl, axis)] if lo else []) + [ap] + ([np.expand_dims(hh, axis)] if hi else [])
    r = np.moveaxis(oracle.KERNELS[op](np.moveaxis(np.concatenate(parts, axis=axis), axis, -1)), -1, axis)
    return (r if post is None else r / post).astype(a.dtype)


# ---------------------------------------------------------------------------------------------- stencil2
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_stencil2_sweep(dtype):
    """Field, out=, metrics and halo planes each on their own offset; every op, shift, boundary and metric layout."""
    from xgcm_b200 import ops

    offs = _offsets(dtype)
    k = 0
    with _Capture("stencil2"):
        for si, shape in enumerate(_stencil_shapes(dtype)):
            a = _field(shape, dtype, 100 + si)
            for axis, op in itertools.product(range(len(shape)), OPS):
                # every boundary and shift with a rotating metric layout, then every metric layout with each
                # length-preserving shift (the forms the TMA, tile and z-batched kernels take)
                cases = [(s, b, None, None) for s, b in itertools.product(SHIFTS, BCS)]
                cases += [(s, BCS[(i + j) % len(BCS)], m, al) for j, s in enumerate(SHIFTS[:2])
                          for i, m in enumerate(METRICS) for al in (True, False)]
                for (lo, hi), (bc, fill), layout, aligned in cases:
                    if shape[axis] + lo + hi - 1 <= 0 or (bc == "extrapolate" and shape[axis] < 2):
                        continue
                    pk, qk = layout or METRICS[k % len(METRICS)]
                    o_in, o_out, o_m = offs[k % len(offs)], offs[(k // 2) % len(offs)], offs[(k // 3) % len(offs)]
                    if aligned:  # the staged kernels want every pointer aligned
                        o_in = o_out = o_m = 0
                    elif aligned is False and o_in == o_out == o_m == 0:
                        o_in = offs[-1]
                    halo = (lo or hi) and k % 5 == 4
                    k += 1
                    oshape = list(shape)
                    oshape[axis] += lo + hi - 1
                    pre = _metric(_layout(pk, shape), dtype, k)
                    post = _metric(_layout(qk, oshape), dtype, k + 1)
                    out = _empty(oshape, dtype, o_out)
                    ctx = f"{shape} axis={axis} {op} ({lo},{hi}) {bc} pre={pk} post={qk} off=({o_in},{o_out},{o_m})"
                    if halo:
                        plane = [s for d, s in enumerate(shape) if d != axis]
                        hl = _field(plane, dtype, k + 2) if lo else None
                        hh = _field(plane, dtype, k + 3) if hi else None
                        ops.stencil2(_dev(a, o_in), axis, op, lo, hi, None, 0.0, pre=_dev(pre, o_m),
                                     post=_dev(post, o_m), halo_lo=_dev(hl, o_m), halo_hi=_dev(hh, o_out), out=out)
                        want = _oracle(_halo_want, op, a, axis, lo, hi, pre, post, hl, hh)
                        _eq(out, want, "halo " + ctx)
                        continue
                    ops.stencil2(_dev(a, o_in), axis, op, lo, hi, bc if (lo or hi) else None, fill,
                                 pre=_dev(pre, o_m), post=_dev(post, o_m), out=out)
                    want = _oracle(oracle.stencil2, op, a, axis, lo, hi, bc if (lo or hi) else None, fill, pre, post)
                    _eq(out, want.astype(dtype), ctx)


# ---------------------------------------------------------------------------------------------- stencil_multi
def _multi_orders(nd):
    """Ordered chains of 2 and 3 of the last three dims; on a 4-D field also the chains of dims 0..2, which leave
    the innermost dim alone."""
    dims = list(range(max(0, nd - 3), nd))
    orders = [p for r in (2, 3) for p in itertools.permutations(dims, r)]
    if nd >= 4:
        orders += list(itertools.permutations(range(3), 3))
    return orders


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_stencil_multi_sweep(dtype):
    """Every application order of 2 and 3 axes (innermost first takes the TMA kernel when it can, every other order
    the marching kernel), every op, shifts and boundaries per axis, on aligned and misaligned fields."""
    from xgcm_b200 import ops

    offs = _offsets(dtype)
    k = 0
    with _Capture("stencil_multi"):
        for si, shape in enumerate([(4, 6, 520), (4, 6, 517), (3, 5, 136), (3, 5, 12), (2, 3, 5, 16), (6, 2, 8)]):
            a = _field(shape, dtype, 200 + si)
            for order, op in itertools.product(_multi_orders(len(shape)), OPS):
                # first every length-preserving combination (the form the TMA kernel takes), then two mixed ones
                los = list(itertools.product((0, 1), repeat=len(order)))
                for rep in range(len(los) + 2):
                    specs = []
                    for j, ax in enumerate(order):
                        lo, hi = (los[rep][j], 1 - los[rep][j]) if rep < len(los) else SHIFTS[(k + j + rep) % 4]
                        bc, fill = BCS3[(k + 2 * j) % len(BCS3)]
                        specs.append((ax, op, lo, hi, bc if (lo or hi) else None, fill))
                    # aligned and misaligned in turn (the TMA kernel wants an aligned field)
                    off = 0 if rep % 2 == 0 else offs[1 + k % (len(offs) - 1)]
                    k += 1
                    got = ops.stencil_multi(_dev(a, off), specs)
                    want = a
                    for ax, op_, lo, hi, bc, fill in specs:
                        want = _oracle(oracle.stencil2, op_, want, ax, lo, hi, bc, fill)
                    _eq(got, want, f"{shape} {specs} off={off}")


# ---------------------------------------------------------------------------------------------- stencil_pair
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_stencil_pair_sweep(dtype):
    """Both operators of every op pair, subtract modes, metrics present or not, aligned or misaligned operands."""
    from xgcm_b200 import ops

    offs = _offsets(dtype)
    k = 0
    with _Capture("stencil_pair"):
        for si, shape in enumerate([(4, 6, 520), (4, 6, 517), (3, 5, 136), (3, 5, 12), (2, 3, 5, 16)]):
            a = _field(shape, dtype, 300 + si)
            b = _field(shape, dtype, 310 + si)
            for axis_b, (op_a, op_b), met in itertools.product(range(len(shape) - 1), itertools.product(OPS, OPS),
                                                                (True, False)):
                for aligned in (True, False):
                    la, lb = k % 2, (k // 2) % 2
                    (bca, fa), (bcb, fb) = BCS3[k % len(BCS3)], BCS3[(k + 2) % len(BCS3)]
                    c = k // 4  # one step per (op pair, axis): every layout meets both aligned and misaligned operands
                    pa = _metric(_layout([None, "lead1", "full", "first"][c % 4], shape), dtype, k)
                    pb = _metric(_layout(["lead1", None, "first", "full"][(c // 4) % 4], shape), dtype, k + 1)
                    post = _metric(_layout([None, "lead1", "first", "last"][(c // 2) % 4], shape), dtype, k + 2)
                    if not met:
                        pa = pb = post = None
                    elif pa is None and pb is None and post is None:
                        post = _metric(_layout("lead1", shape), dtype, k + 3)
                    sub = k % 3
                    oa, ob, om = (0, 0, 0) if aligned else (offs[1 + k % (len(offs) - 1)], offs[k % len(offs)],
                                                            offs[(k // 3) % len(offs)])
                    k += 1
                    got = ops.stencil_pair(_dev(a, oa), _dev(b, ob), (op_a, la, 1 - la, bca, fa),
                                           (axis_b, op_b, lb, 1 - lb, bcb, fb), sub, pre_a=_dev(pa, om),
                                           pre_b=_dev(pb, om), post=_dev(post, om))
                    want = _oracle(oracle.stencil_pair, op_a, a, len(shape) - 1, la, 1 - la, bca, fa, pa, op_b, b,
                                   axis_b, lb, 1 - lb, bcb, fb, pb, sub, post)
                    _eq(got, want, f"{shape} {op_a}/{op_b} axis_b={axis_b} sub={sub} off=({oa},{ob},{om})")
        # the staged tile kernel of the pair, every diff / interp pair with per-level (full, dz) and shared metrics
        shape = (4, 6, 520)
        a, b = _field(shape, dtype, 320), _field(shape, dtype, 321)
        for (op_a, op_b), (ka, kb, kp) in itertools.product(
                itertools.product(("diff", "interp"), repeat=2),
                [("full", None, None), (None, "first", None), (None, None, "first"), ("lead1", "lead1", "lead1")]):
            pa, pb, post = (_metric(_layout(m, shape), dtype, i) for i, m in enumerate((ka, kb, kp)))
            got = ops.stencil_pair(_dev(a), _dev(b), (op_a, 1, 0, "periodic", 0.0), (1, op_b, 0, 1, "fill", 0.0), 0,
                                   pre_a=_dev(pa), pre_b=_dev(pb), post=_dev(post))
            want = _oracle(oracle.stencil_pair, op_a, a, 2, 1, 0, "periodic", 0.0, pa, op_b, b, 1, 0, 1, "fill", 0.0,
                           pb, 0, post)
            _eq(got, want, f"tile pair {op_a}/{op_b} metrics=({ka},{kb},{kp})")


# ---------------------------------------------------------------------------------------------- cumscan
def _cumscan_cases():
    seen = []
    for table, rev in ((oracle.CUMSUM_TABLE_FWD, False), (oracle.CUMSUM_TABLE_REV, True)):
        for trim, (plo, phi) in table.values():
            if (rev, trim, plo, phi) not in seen:
                seen.append((rev, trim, plo, phi))
    return seen


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_cumscan_sweep(dtype):
    """Rows (narrow and 16-byte tiled), strided columns either side of the vector switch; metrics, skipna, offsets."""
    from xgcm_b200 import ops

    offs = _offsets(dtype)
    shapes = [((37, 776), 1), ((37, 775), 1), ((3, 2, 1032), 2), ((5, 40), 1), ((6, 20, 36), 0), ((6, 20, 36), 1),
              (((40, 48, 704) if dtype == np.float32 else (40, 24, 704)), 0), ((40, 48, 700), 0), ((70, 1, 5), 0)]
    k = 0
    with _Capture("cumscan"):
        for si, (shape, axis) in enumerate(shapes):
            a = _field(shape, dtype, 400 + si)
            for (rev, trim, plo, phi), (bc, fill) in zip(_cumscan_cases() * 2, BCS3 * 4):
                oshape = list(shape)
                oshape[axis] = shape[axis] - (0 if trim == "none" else 1) + plo + phi
                pre = _metric(_layout([None, "lead1", "full", "last"][k % 4], shape), dtype, k)
                post = _metric(_layout([None, "first", "lead1", "nolast"][(k // 2) % 4], oshape), dtype, k + 1)
                skipna = k % 3 != 2
                off = offs[k % len(offs)]
                om = offs[(k // 2) % len(offs)]
                k += 1
                got = ops.cumscan(_dev(a, off), axis, rev, trim, plo, phi, bc, fill, _dev(pre, om), _dev(post, om),
                                  skipna)
                want = _oracle(oracle.cumscan, a, axis, rev, trim, plo, phi, bc if (plo or phi) else None, fill, pre,
                               post, skipna)
                _eq(got, want.astype(dtype), f"{shape} axis={axis} rev={rev} {trim} ({plo},{phi}) {bc} off={off}")


# ---------------------------------------------------------------------------------------------- wreduce
def _fsum_bound_check(got, a, w, axis, mode, skipna, ctx):
    """Row reductions accumulate in fp64 and round once: within 1/2 ulp of the exact sum of the products rounded
    to the field dtype, plus the fp64 accumulation error (n - 1) 2^-53 sum |p_i| (for the mean, of both sums)."""
    dt = a.dtype.type
    am = np.moveaxis(a, axis, -1)
    wm = np.ones_like(am) if w is None else np.moveaxis(np.broadcast_to(w, a.shape), axis, -1).astype(a.dtype)
    rows, wrows = am.reshape(-1, am.shape[-1]), wm.reshape(-1, am.shape[-1])
    g = np.asarray(got).reshape(-1)
    n = rows.shape[1]
    eps = 2.0 ** -53
    for r in range(rows.shape[0]):
        x, ww = rows[r], wrows[r]
        with np.errstate(all="ignore"):
            p = (x * ww).astype(dt)
        if mode == "sum":
            p = p[~np.isnan(p)] if skipna else p
            if not np.all(np.isfinite(p)):
                want = dt(np.sum(p.astype(np.float64)))
                assert np.array_equal(g[r], want, equal_nan=True), f"{ctx} row {r}: {g[r]} != {want}"
                continue
            exact = math.fsum(float(v) for v in p)
            bound = (max(n - 1, 0)) * eps * float(np.sum(np.abs(p.astype(np.float64))))
        else:
            valid = ~np.isnan(x) if skipna else np.ones(n, bool)
            p, wv = p[valid], ww[valid]
            den = math.fsum(float(v) for v in wv)
            if den == 0 or not np.all(np.isfinite(p)):  # NaN (0 / 0, a NaN kept by skipna=False) or +-inf
                with np.errstate(all="ignore"):
                    want = dt(np.sum(p.astype(np.float64)) / den) if den != 0 else dt(np.nan)
                assert np.array_equal(g[r], want, equal_nan=True), f"{ctx} row {r}: {g[r]} != {want}"
                continue
            num = math.fsum(float(v) for v in p)
            exact = num / den
            acc = max(n - 1, 0) * eps
            bound = (acc * float(np.sum(np.abs(p.astype(np.float64)))) + abs(exact) * acc * float(np.sum(np.abs(wv)))) \
                / abs(den) + abs(exact) * 2.0 ** -52
        ulp = float(np.spacing(dt(max(abs(exact), abs(float(g[r]))))))
        err = abs(float(g[r]) - exact)
        assert err <= 0.5 * ulp + bound, f"{ctx} row {r}: got {g[r]!r}, exact {exact!r}, err {err} > {0.5 * ulp + bound}"


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_wreduce_sweep(dtype):
    """Strided reductions bit-exact against numpy either side of the vector switch; row reductions (vector and
    scalar loads, misaligned rows) against an exact sum."""
    from xgcm_b200 import ops

    offs = _offsets(dtype)
    strided = [((40, 48, 704), 0), ((40, 48, 700), 0), ((22, 30, 1536), 1), ((30, 12, 40), 1), ((30, 12, 40), 0)]
    k = 0
    with _Capture("wreduce"):
        for si, (shape, axis) in enumerate(strided):
            a = _field(shape, dtype, 500 + si)
            level = tuple(n if d == axis else 1 for d, n in enumerate(shape))
            for wshape, mode, skipna in itertools.product((None, shape, (1,) + shape[1:], level), ("sum", "mean"),
                                                          (True, False)):
                w = _metric(wshape, dtype, k)
                off = offs[k % len(offs)]
                k += 1
                got = ops.wreduce(_dev(a, off), axis, _dev(w, offs[(k // 2) % len(offs)]), mode, skipna)
                _eq(got, _oracle(oracle.wreduce, a, w, axis, mode, skipna), f"{shape} axis={axis} w={wshape} {mode}")
        for si, shape in enumerate([(7, 9, 1000), (7, 9, 999), (3, 1), (5, 64)]):
            a = _field(shape, dtype, 550 + si, specials=False)
            a.reshape(-1)[a.size // 2] = np.nan
            for wk, mode, skipna in itertools.product((None, "last", "full"), ("sum", "mean"), (True, False)):
                w = _metric(_layout(wk, shape), dtype, k)
                off = offs[k % len(offs)]
                k += 1
                got = ops.wreduce(_dev(a, off), -1, _dev(w, offs[(k // 2) % len(offs)]), mode, skipna).cpu().numpy()
                _fsum_bound_check(got, a, w, len(shape) - 1, mode, skipna, f"{shape} w={wk} {mode} skipna={skipna}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_row_reduction_against_exact_sum(dtype):
    """k_reduce_rows rounds once: rows of 1 to 10^6 cells, and mixed-sign rows whose sum cancels to a few ulp of the
    terms, sum and mean, with and without weights, skipna both ways."""
    from xgcm_b200 import ops

    rng = np.random.default_rng(570)
    with _Capture("wreduce"):
        for n in (1, 2, 3, 31, 1000, 4097, 1_000_000):
            rows = 3 if n < 1_000_000 else 1
            a = (rng.standard_normal((rows, n)) * 10.0 ** rng.integers(-3, 4, size=(rows, n))).astype(dtype)
            if n >= 4:  # heavy cancellation: a copy of the first half with its sign flipped, plus a tiny tail
                h = n // 2
                a[-1, h:2 * h] = -a[-1, :h][::-1]
                a[-1, -1] = dtype(1e-3)
            if n >= 3:
                a[0, 1] = np.nan
            w = _metric((1, n), dtype, n)
            for weight, mode, skipna in itertools.product((None, w), ("sum", "mean"), (True, False)):
                got = ops.wreduce(_dev(a, n % len(_offsets(dtype))), 1, _dev(weight), mode, skipna).cpu().numpy()
                _fsum_bound_check(got, a, weight, 1, mode, skipna, f"n={n} w={weight is not None} {mode} {skipna}")


# ---------------------------------------------------------------------------------------------- vinterp
def _extreme_columns(dtype, ncol, seed):
    """Columns whose dy spans 10^+-12, with zero slopes, NaNs, a dy that overflows to +-inf and a subnormal dy."""
    rng = np.random.default_rng(seed)
    n = 5
    phi = (rng.standard_normal((n, ncol)) * 10.0 ** rng.integers(-12, 12, size=(n, ncol))).astype(dtype)
    phi[:, :50] = 0.0
    phi[2, 50:80] = np.nan
    phi[1, 100:200] = phi[2, 100:200]  # dy == 0
    big = np.finfo(dtype).max
    tiny = np.finfo(dtype).smallest_subnormal
    phi[1, 200:210], phi[2, 200:210] = big, -big  # dy overflows to -inf
    phi[1, 210:220], phi[2, 210:220] = -big, big  # to +inf
    phi[1, 220:230], phi[2, 220:230] = 0.0, tiny * 3  # subnormal dy
    phi[1, 230:240], phi[2, 230:240] = tiny, -tiny
    theta = np.array([0.1, 0.7, 1.9, 3.0000001, 7.3], dtype=dtype).reshape(n, 1)
    target = np.array([0.05, 0.1, 0.33, 0.7000001, 1.0, 1.3, 2.5, 3.0, 3.5, 7.0, 7.3, 9.0], dtype=dtype)
    return phi, theta, target


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_vinterp_sweep(dtype):
    """Shared theta and theta fields, TMA-sized and small, aligned and misaligned phi; extreme slopes on every route;
    the conservative remap."""
    from xgcm_b200 import ops

    offs = _offsets(dtype)
    k = 0
    with _Capture("vinterp"):
        for ncol in (4096, 4093, 300, 20):
            phi, theta, target = _extreme_columns(dtype, ncol, 600 + ncol)
            for off in offs:
                for mask, bypass in ((True, False), (False, False), (True, True)):
                    want = _oracle(oracle.vinterp_linear, phi, np.broadcast_to(theta, phi.shape), target, 0, mask,
                                   bypass)
                    got = ops.vinterp_linear(_dev(phi, off), _dev(theta), _dev(target), 0, mask, bypass)
                    _eq(got, want, f"shared ncol={ncol} off={off} mask={mask} bypass={bypass}")
                    thf = np.ascontiguousarray(np.broadcast_to(theta, phi.shape)) * (1 + 0.01 * (k % 3))
                    thf = thf.astype(dtype)
                    k += 1
                    want = _oracle(oracle.vinterp_linear, phi, thf, target, 0, mask, bypass)
                    got = ops.vinterp_linear(_dev(phi, off), _dev(thf, off), _dev(target), 0, mask, bypass)
                    _eq(got, want, f"field ncol={ncol} off={off} mask={mask} bypass={bypass}")
        # 200 levels and 40 targets: too many for two columns per lane in shared memory (one-column TMA kernel)
        rng = np.random.default_rng(60)
        phi = _field((200, 512), dtype, 63)
        theta = np.cumsum(0.1 + rng.random(200)).astype(dtype).reshape(200, 1)
        target = np.linspace(-1, float(theta[-1, 0]) + 1, 40).astype(dtype)
        for off in offs:
            want = _oracle(oracle.vinterp_linear, phi, np.broadcast_to(theta, phi.shape), target, 0, True)
            _eq(ops.vinterp_linear(_dev(phi, off), _dev(theta), _dev(target), 0, True), want, f"200 levels off={off}")
        rng = np.random.default_rng(61)
        for shape, axis in (((20, 6, 37), 0), ((3, 25, 40), 1), ((12, 64), 0)):
            phi = _field(shape, dtype, 62, specials=False)
            n = shape[axis]
            bshape = [n if d == axis else s for d, s in enumerate(shape)]
            bshape[axis] = n + 1
            theta = np.cumsum(0.1 + rng.random(bshape), axis=axis).astype(dtype)
            bins = np.linspace(float(theta.min()) - 0.5, float(theta.max()) + 0.5, 9).astype(dtype)
            for off in offs:
                for tb in (bins, bins[::-1].copy()):
                    got = ops.vinterp_conservative(_dev(phi, off), _dev(theta, off), _dev(tb), axis)
                    _eq(got, _oracle(oracle.vinterp_conservative, phi, theta, tb, axis), f"conservative {shape} off={off}")


# ---------------------------------------------------------------------------------------------- elementwise
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_elementwise_sweep(dtype):
    """pad (rows and general), binary (every operator, vector and scalar), fill_uniform, fold_rows, strided copies."""
    from xgcm_b200 import ops

    offs = _offsets(dtype)
    k = 0
    with _Capture("elementwise"):
        for si, shape in enumerate([(7, 1027), (3, 5, 130), (4, 6, 12), (2, 3, 4, 33), (4099,)]):
            a = _field(shape, dtype, 700 + si)
            for axis in range(len(shape)):
                for (lo, hi), (bc, fill) in itertools.product([(1, 0), (0, 1), (1, 1), (3, 2)], BCS):
                    if (bc == "periodic" and max(lo, hi) > shape[axis]) or (bc == "extrapolate" and max(lo, hi) > 1):
                        continue
                    off = offs[k % len(offs)]
                    k += 1
                    got = ops.pad(_dev(a, off), axis, lo, hi, bc, fill)
                    _eq(got, _oracle(oracle.pad_axis, a, axis, lo, hi, bc, fill), f"pad {shape} {axis} {bc} off={off}")
        fns = {"mul": np.multiply, "div": np.true_divide, "add": np.add, "sub": np.subtract,
               "divnz": lambda x, y: np.where(y != 0, x / np.where(y != 0, y, 1), np.nan).astype(x.dtype)}
        for ashape, bshape in (((3, 4, 6, 8), (1, 4, 1, 8)), ((3, 4, 6, 8), (3, 4, 6, 8)), ((5, 7), (5, 1)),
                               ((6, 130), (130,))):
            x = _field(ashape, dtype, 710)
            y = _field(bshape, dtype, 711)
            y.reshape(-1)[::5] = 0.0
            for name, fn in fns.items():
                for off in offs:
                    got = ops.binary(name, _dev(x, off), _dev(y, offs[(off + 1) % len(offs)]))
                    _eq(got, _oracle(fn, x, y).astype(dtype), f"binary {name} {ashape} {bshape} off={off}")
        for off in offs:
            got = ops.fill_uniform(_empty((10_003,), dtype, off), seed=5, offset=off)
            _eq(got, ops.fill_uniform_host(np.empty(10_003, dtype=dtype), seed=5, offset=off), f"fill_uniform {off}")
        # north-fold rows: out[.., r, .., k, ..] = +-(x * pre)[.., n - 1 - skip - r, .., (mirror - k) mod period, ..]
        x = _field((3, 9, 16), dtype, 720)
        pre = _metric((1, 9, 16), dtype, 721)
        for (width, skip, mirror, negate), off in itertools.product([(1, 0, 15, False), (2, 1, 16, True)], offs):
            got = ops.fold_rows(_dev(x, off), 1, 2, width, skip, mirror, 16, negate, pre=_dev(pre, off))
            src = (x * pre)[:, [9 - 1 - skip - r for r in range(width)], :][:, :, [(mirror - c) % 16 for c in range(16)]]
            _eq(got, (-src if negate else src).astype(dtype), f"fold_rows w={width} off={off}")
        # strided copies: a flipped and a transposed edge into a padded buffer
        src = _field((6, 8), dtype, 730)
        for off in offs:
            dst = _empty((8, 10), dtype, off)
            ts = _dev(src, offs[-1 - offs.index(off)])
            ops.strided_copy(dst, 11, [10, 1], ts, 7, [-1, 8], [6, 6], negate=True)
            want = np.full((8, 10), SENTINEL, dtype=dtype)
            want.reshape(-1)[[11 + 10 * i + j for i in range(6) for j in range(6)]] = \
                -src.reshape(-1)[[7 - i + 8 * j for i in range(6) for j in range(6)]]
            _eq(dst, want, f"strided_copy off={off}")
            dst2 = _empty((8, 10), dtype, off)
            ops.strided_copy_batch([(dst2, 0, [1, 10], ts, 0, [8, 1], [6, 8], False),
                                    (dst2, 79, [10, -1], ts, 40, [8, 1], [1, 4], True)])
            want = np.full((8, 10), SENTINEL, dtype=dtype)
            want.reshape(-1)[[i + 10 * j for i in range(6) for j in range(8)]] = src.reshape(-1)
            want.reshape(-1)[[79 - i for i in range(4)]] = -src.reshape(-1)[40:44]
            _eq(dst2, want, f"strided_copy_batch off={off}")


# ---------------------------------------------------------------------------------------------- host twins
@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_host_twins_sweep(dtype):
    """The slab pipelines hand the kernels plane offsets that are only element aligned when a plane is not a
    multiple of 16 bytes: (9, 33, 70) fp32 makes every slab after the first misaligned."""
    from xgcm_b200 import ops

    with _Capture("host"):
        for si, shape in enumerate([(9, 33, 70), (9, 33, 64), (5, 7, 513)]):
            a = _field(shape, dtype, 800 + si)
            dx = _metric((1,) + shape[1:], dtype, 801)
            dz = _metric((shape[0], 1, 1), dtype, 802)
            for axis, op, ((lo, hi), (bc, fill)) in itertools.product(range(3), OPS, zip(SHIFTS, BCS)):
                pre, post = (dz, dx if lo + hi == 1 else None) if (axis + si) % 2 else (None, None)
                if axis == 0 and bc == "periodic":  # the slab pipeline takes no pre-metric there
                    pre = None
                got = ops.stencil2_host(a, axis, op, lo, hi, bc if (lo or hi) else None, fill, pre=pre, post=post)
                want = _oracle(oracle.stencil2, op, a, axis, lo, hi, bc if (lo or hi) else None, fill, pre, post)
                _eq(got, want.astype(dtype), f"stencil2_host {shape} {axis} {op}")
            specs = [(2, "diff", 1, 0, "periodic", 0.0), (1, "interp", 0, 1, "fill", 1.5), (0, "max", 0, 1, "extend", 0.0)]
            for got, (ax, op, lo, hi, bc, fill) in zip(ops.stencil2_host_multi(a, specs), specs):
                _eq(got, _oracle(oracle.stencil2, op, a, ax, lo, hi, bc, fill), f"stencil2_host_multi {shape} {ax}")
            for axis, (rev, trim, plo, phi) in itertools.product(range(3), _cumscan_cases()[::3]):
                got = ops.cumscan_host(a, axis, rev, trim, plo, phi, "extend", 0.0, pre=dx)
                want = _oracle(oracle.cumscan, a, axis, rev, trim, plo, phi, "extend" if (plo or phi) else None, 0.0, dx)
                _eq(got, want.astype(dtype), f"cumscan_host {shape} {axis}")
            for axis in range(2):
                got = ops.wreduce_host(a, axis, dz if axis == 0 else dx, "sum", True)
                _eq(got, _oracle(oracle.wreduce, a, dz if axis == 0 else dx, axis, "sum", True), f"wreduce_host {axis}")
            got = ops.wreduce_host(a, 2, dx, "mean", True)
            _fsum_bound_check(got, a, dx, 2, "mean", True, f"wreduce_host rows {shape}")
            th = np.cumsum(0.5 + np.random.default_rng(803).random(shape[0])).astype(dtype)
            tg = np.linspace(0, float(th[-1]) + 1, 7).astype(dtype)
            got = ops.vinterp_linear_host(a, th.reshape(-1, 1, 1), tg, 0, True)
            _eq(got, _oracle(oracle.vinterp_linear, a, np.broadcast_to(th.reshape(-1, 1, 1), shape), tg, 0, True),
                f"vinterp_linear_host {shape}")


# ---------------------------------------------------------------------------------------------- Grid on time slices
def _slice_grid(nz, ny, nx, dtype):
    """A C-grid (Z, Y, X) dataset with dx / dy / area at every horizontal position and dz, all of the field dtype."""
    import xgcm_b200 as xg

    rng = np.random.default_rng(900)
    coords = {"Z": np.arange(nz) + 0.5, "Zl": np.arange(nz) + 0.0, "YC": np.arange(ny) + 0.5, "YG": np.arange(ny) + 0.0,
              "XC": np.arange(nx) + 0.5, "XG": np.arange(nx) + 0.0,
              "dz": (("Z",), (1 + rng.random(nz)).astype(dtype)), "dzl": (("Zl",), (1 + rng.random(nz)).astype(dtype))}
    metrics = {("X",): [], ("Y",): [], ("X", "Y"): [], ("Z",): ["dz", "dzl"]}
    for y in ("YC", "YG"):
        for x in ("XC", "XG"):
            for name, key in (("dx", ("X",)), ("dy", ("Y",)), ("ra", ("X", "Y"))):
                coords[f"{name}_{y}{x}"] = ((y, x), (0.5 + rng.random((ny, nx))).astype(dtype))
                metrics[key].append(f"{name}_{y}{x}")
    ds = xg.Dataset(coords=coords)
    grid = xg.Grid(ds, coords={"X": {"center": "XC", "left": "XG"}, "Y": {"center": "YC", "left": "YG"},
                               "Z": {"center": "Z", "left": "Zl"}},
                   padding={"X": "periodic", "Y": "fill", "Z": "extend"}, metrics=metrics, autoparse_metadata=False)
    return ds, grid


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(4, 5, 7, 9), (4, 4, 6, 520)])
def test_grid_ops_on_misaligned_time_slices(dtype, shape):
    """x[1], x[2], x[3] of a device (T, Z, Y, X) field through the Grid: equal bit for bit to the same call on
    x[t].clone(), and to the oracle where it restates the op.  (4, 5, 7, 9): Z Y X is odd, so the slices sit 1, 2 and
    3 elements past a 16-byte boundary (fp32).  (4, 4, 6, 520): X is TMA-sized; the field is cut from its allocation
    one element in, so every slice is misaligned while its clone takes the staged kernels."""
    import torch

    import xgcm_b200 as xg

    with _Capture("grid"):
        _, nz, ny, nx = shape
        ds, grid = _slice_grid(nz, ny, nx, dtype)
        a = _field(shape, dtype, 901, specials=False)
        a[1, 0, 0, 0] = np.nan
        base = torch.empty(a.size + 2, dtype=_tdt(dtype), device=DEV)
        x = base[1:1 + a.size].view(shape)
        x.copy_(torch.from_numpy(a))
        b = _dev(_field(shape, dtype, 902, specials=False), 1)
        dz = ds["dz"].values
        dx = ds["dx_YCXC"].values
        levels = np.linspace(-0.5, nz + 0.5, 7)
        pos = {"c": ("Z", "YC", "XC"), "u": ("Z", "YC", "XG"), "v": ("Z", "YG", "XC")}

        def calls(f, g):
            c = lambda t: xg.DataArray(t, dims=pos["c"])  # noqa: E731
            u = lambda t: xg.DataArray(t, dims=pos["u"])  # noqa: E731
            v = lambda t: xg.DataArray(t, dims=pos["v"])  # noqa: E731
            out = {}
            for ax in ("X", "Y", "Z"):
                for op in ("diff", "interp", "min", "max"):
                    out[f"{op} {ax}"] = getattr(grid, op)(c(f), ax)
                out[f"derivative {ax}"] = grid.derivative(c(f), ax)
                out[f"cumsum {ax}"] = grid.cumsum(c(f), ax)
                out[f"cumint {ax}"] = grid.cumint(c(f), ax)
                out[f"integrate {ax}"] = grid.integrate(c(f), ax)
                out[f"average {ax}"] = grid.average(c(f), ax)
            out["interp metric X"] = grid.interp(c(f), "X", metric_weighted=["X", "Y"])
            out["interp XYZ"] = grid.interp(c(f), ["X", "Y", "Z"])
            out["divergence"] = grid.divergence(u(f), v(g))
            out["vorticity"] = grid.vorticity(u(f), v(g))
            out["transform linear"] = grid.transform(c(f), "Z", levels)
            return out

        for t in (1, 2, 3):
            xt = x[t]
            assert xt.data_ptr() % 16 == ((1 + t * nz * ny * nx) * a.itemsize) % 16
            sliced, cloned = calls(xt, b[t]), calls(xt.clone(), b[t].clone())
            for name, got in sliced.items():
                _eq(got.values, cloned[name].values, f"t={t} {name}: slice vs clone")
            at = a[t]
            for ax, i, bc in (("X", 2, "periodic"), ("Y", 1, "fill"), ("Z", 0, "extend")):
                for op in ("diff", "interp", "min", "max"):
                    _eq(sliced[f"{op} {ax}"].values, _oracle(oracle.stencil2, op, at, i, 1, 0, bc, 0.0), f"t={t} {op} {ax}")
            _eq(sliced["derivative X"].values, _oracle(oracle.stencil2, "diff", at, 2, 1, 0, "periodic", 0.0, None,
                                                       ds["dx_YCXG"].values[None]), f"t={t} derivative X")
            _eq(sliced["integrate Z"].values, _oracle(oracle.wreduce, at, dz[:, None, None], 0), f"t={t} integrate Z")
            _fsum_bound_check(sliced["integrate X"].values, at, dx[None], 2, "sum", True, f"t={t} integrate X")
            want = at
            for i, bc in ((2, "periodic"), (1, "fill"), (0, "extend")):
                want = _oracle(oracle.stencil2, "interp", want, i, 1, 0, bc, 0.0)
            _eq(sliced["interp XYZ"].values, want, f"t={t} interp XYZ")
            _eq(sliced["transform linear"].values,
                _oracle(oracle.vinterp_linear, at, np.broadcast_to(ds["Z"].values[:, None, None], at.shape), levels, 0, True),
                f"t={t} transform")
        # conservative transform: cell bounds on the outer Z position, both slices of fields cut one element in
        bounds = np.cumsum(0.5 + np.random.default_rng(903).random((shape[0], nz + 1, ny, nx)), axis=1).astype(dtype)
        th = _dev(bounds, 1)
        dsc = xg.Dataset(coords={"z": np.arange(nz) + 0.5, "zo": np.arange(nz + 1.0)})
        gc = xg.Grid(dsc, coords={"Z": {"center": "z", "outer": "zo"}}, autoparse_metadata=False)
        bins = np.linspace(0, float(bounds.max()) + 1, 6).astype(dtype)
        for t in (1, 2, 3):
            q = lambda f: xg.DataArray(f, dims=("z", "y", "x"))  # noqa: E731
            s = lambda f: xg.DataArray(f, dims=("zo", "y", "x"), name="sig")  # noqa: E731
            got = gc.transform(q(x[t]), "Z", bins, target_data=s(th[t]), method="conservative")
            ref = gc.transform(q(x[t].clone()), "Z", bins, target_data=s(th[t].clone()), method="conservative")
            _eq(got.values, ref.values, f"t={t} conservative: slice vs clone")
            _eq(got.values, _oracle(oracle.vinterp_conservative, a[t], bounds[t], bins, 0), f"t={t} conservative")


# ---------------------------------------------------------------------------------------------- coverage
_SWEEPS = {"stencil2", "stencil_multi", "stencil_pair", "cumscan", "wreduce", "vinterp", "elementwise", "host", "grid"}


@pytest.mark.gpu
def test_every_instance_ran():
    """(manifest) - (launched by the sweeps above) == ALLOWLIST.  Runs last; needs the whole file."""
    missing = _SWEEPS - set(_LAUNCHED)
    if missing:
        pytest.skip(f"the sweeps {sorted(missing)} did not run in this session")
    _, entries = _manifest()
    compiled = {_key(n) for _, n in entries}
    launched = set().union(*_LAUNCHED.values())
    uncovered = compiled - launched - set(ALLOWLIST)
    stale = set(ALLOWLIST) - compiled
    ran_anyway = set(ALLOWLIST) & launched
    by_template = defaultdict(list)
    for k in sorted(uncovered):
        by_template[k.split("<")[0]].append(k)
    report = "\n".join(f"  {t} ({len(v)}):\n    " + "\n    ".join(v) for t, v in sorted(by_template.items()))
    assert not uncovered, f"{len(uncovered)} compiled instances never ran against the oracle:\n{report}"
    assert not stale and not ran_anyway, (stale, ran_anyway)
