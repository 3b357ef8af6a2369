"""Every kind of memory a caller may hand the C ABI, bit for bit.

The pointers include/sicp_b200.h marks [h|d] may be host or device memory, and clouds of 4 MiB or
more in pageable host memory go through the threaded staging of csrc/upload.cu.  Here every such
pointer gets each of these kinds:

  P    pageable NumPy                          P+   pageable, offset by one element
  H    pinned (torch pin_memory) NumPy         D    a CUDA tensor
  D+   a CUDA view offset by one element: 8 bytes for float64 and int64, 4 for float32, 1 for uint8

and clouds also these three, which `_capi._as_f64_xyz` converts before the call:

  T    a CPU torch tensor                      D32  a float32 CUDA tensor
  DT   a non-contiguous CUDA tensor, (3, n).T

Every result is compared BIT FOR BIT with the same call made from P with option upload_threads 0
(the driver's own staging) on the same engine; the inputs of the converted kinds are compared
with a P baseline of the same converted float64 values.  The library is deterministic run to run.

The transform is also checked against exact rational arithmetic (test_transform_rounds_like_its_expression).
"""
import ctypes as C
import zlib
from fractions import Fraction

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from conftest import load_pair

import simpleicp_b200 as sb
from simpleicp_b200 import _capi, pointcloud, synthetic

pytestmark = pytest.mark.gpu

KINDS = ("P", "P+", "H", "D", "D+")
CLOUD_KINDS = KINDS + ("T", "D32", "DT")
TORCH = {np.dtype(np.float64): torch.float64, np.dtype(np.float32): torch.float32,
         np.dtype(np.int64): torch.int64, np.dtype(np.uint8): torch.uint8}
SENTINEL = {np.dtype(np.float64): np.nan, np.dtype(np.float32): np.nan, np.dtype(np.int64): -7, np.dtype(np.uint8): 7}


# ---- buffers of each kind ------------------------------------------------------------------------

class Buf:
    """A buffer of one kind holding `shape` elements of `dtype`, filled with a sentinel.  Offset
    kinds are views one element into an allocation with one guard element on each side."""

    def __init__(self, kind, shape, dtype):
        dtype = np.dtype(dtype)
        shape = tuple(int(s) for s in np.atleast_1d(shape))
        n = int(np.prod(shape))
        self.kind, self.shape, self.dtype = kind, shape, dtype
        fill = SENTINEL[dtype]
        if kind in ("P", "P+"):
            self.base = np.full(n + 2, fill, dtype)
            self.obj = self.base[:n].reshape(shape) if kind == "P" else self.base[1:n + 1].reshape(shape)
        elif kind == "H":
            self.base = torch.full((n,), fill, dtype=TORCH[dtype], pin_memory=True)
            self.obj = self.base.numpy().reshape(shape)
        elif kind in ("D", "D+"):
            self.base = torch.full((n + 2,), fill, dtype=TORCH[dtype], device="cuda")
            self.obj = (self.base[:n] if kind == "D" else self.base[1:n + 1]).view(shape)
        else:
            raise ValueError(kind)
        if kind == "D+":  # CUDA allocations are 512-byte aligned: the view is one element off
            assert self.addr % 16 == dtype.itemsize % 16

    @property
    def addr(self) -> int:
        return self.obj.ctypes.data if isinstance(self.obj, np.ndarray) else self.obj.data_ptr()

    def put(self, values):
        values = np.ascontiguousarray(values, dtype=self.dtype).reshape(self.shape)
        if isinstance(self.obj, np.ndarray):
            self.obj[...] = values
        else:
            self.obj.copy_(torch.from_numpy(values))
            torch.cuda.synchronize()
        return self

    def get(self) -> np.ndarray:
        """A host copy; the guard elements of the offset kinds must be untouched."""
        if self.kind in ("P+", "D+"):
            base = _host(self.base)
            guard = base[[0, -1]]
            assert (np.isnan(guard).all() if self.dtype.kind == "f" else (guard == SENTINEL[self.dtype]).all()), \
                f"{self.kind}: a guard element next to the buffer was overwritten"
        return _host(self.obj)


def _host(a) -> np.ndarray:
    if isinstance(a, torch.Tensor):
        return a.detach().cpu().numpy().copy()
    return np.array(a, copy=True)


def _cloud(kind, X):
    """X ((n, 3) float64) in cloud kind `kind` -> (object for the API, the float64 values the library sees)."""
    if kind in KINDS:
        return Buf(kind, X.shape, np.float64).put(X).obj, X
    if kind == "T":
        return torch.from_numpy(X.copy()), X
    if kind == "D32":
        X32 = X.astype(np.float32)
        return torch.from_numpy(X32).cuda(), X32.astype(np.float64)
    if kind == "DT":
        t = torch.from_numpy(np.ascontiguousarray(X.T)).cuda().T
        assert not t.is_contiguous()
        return t, X
    raise ValueError(kind)


def _same(a, b, what):
    """Bit for bit: same dtype, same shape, same bytes (NaN compared as NaN, zeros by sign)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, f"{what}: {a.dtype}{a.shape} vs {b.dtype}{b.shape}"
    if a.tobytes() != b.tobytes():
        bad = np.flatnonzero(((a != b) & ~(np.isnan(a) & np.isnan(b))) if a.dtype.kind == "f" else (a != b))
        pytest.fail(f"{what}: bits differ; {bad.size} of {a.size} values differ, first at {bad[:5].tolist()}")


def _same_all(got: dict, want: dict, what):
    assert got.keys() == want.keys(), f"{what}: {sorted(set(got) ^ set(want))}"
    for k in want:
        _same(got[k], want[k], f"{what}: {k}")


def _seed(*key) -> int:
    return zlib.crc32(repr(key).encode())


@pytest.fixture(scope="module")
def eng(gpu):
    with _capi.Engine() as e:
        yield e


def _options(e, threads=None, chunk_kb=None):
    e.reset_options()
    if threads is not None:
        e.set_option("upload_threads", threads)
    if chunk_kb is not None:
        e.set_option("upload_chunk_kb", chunk_kb)


# ---- a. the exact upload probe -------------------------------------------------------------------

def _probe(e, kind, X, what):
    """Upload the same points twice, as the fixed and as the movable cloud, from two separate
    buffers of `kind`.  set_clouds sends the movable cloud through the foreground upload and the
    fixed cloud through the background upload; every byte of both must arrive.  Without any debug
    hook: every fixed point has its own movable copy at squared distance exactly 0 (a bound of
    1e-300 on the squared distance), every query matches its own index at distance 0 (unit z
    normals), and the identity transform returns the movable cloud itself (rigid_apply with the
    identity is exact up to the sign of zero)."""
    fix, V = _cloud(kind, X)
    mov, _ = _cloud(kind, X)
    n = X.shape[0]
    e.set_clouds(fix, mov)
    e.set_selected(None)
    keep = e.select_in_range(np.eye(4), 1e-150)
    assert keep.all(), f"{what}: {np.count_nonzero(~keep)} fixed points have no exact movable copy"
    one, zero = np.ones(n, np.float32), np.zeros(n, np.float32)
    e.set_normals(zero, zero, one, one)
    idx, d = e.match(np.eye(4))
    bad = np.flatnonzero(idx != np.arange(n))
    assert bad.size == 0, f"{what}: {bad.size} queries do not match their own point, first {bad[:5].tolist()}"
    assert not d.any(), f"{what}: non-zero distances"
    Y = e.transform(np.eye(4))
    assert np.array_equal(Y, V), f"{what}: transform(I) differs from the movable cloud in {np.count_nonzero(Y != V)} values"


# 4 MiB - 16 B (the driver's path), 4 MiB + 8 B (threaded; at 4096 KiB slices the last is 8 bytes),
# exactly three 2 MiB slices and one point more, and 10^6 points (64 KiB slices reuse every staging
# buffer many times)
PROBE_N = (174_762, 174_763, 262_144, 262_145, 1_000_000)


@pytest.mark.parametrize("n", PROBE_N)
@pytest.mark.parametrize("chunk_kb", [64, 100, 2048, 4096])
@pytest.mark.parametrize("threads", [0, 1, 2, 3, 8])
def test_upload_probe(eng, threads, chunk_kb, n):
    assert (3 * 8 * 174_762 < 4 << 20 < 3 * 8 * 174_763) and 3 * 8 * 262_144 == 3 * (2 << 20)
    _options(eng, threads, chunk_kb)
    for kind in CLOUD_KINDS:
        X = np.random.default_rng(_seed(threads, chunk_kb, n, kind)).normal(size=(n, 3)) * 50.0
        _probe(eng, kind, X, f"threads {threads} chunk {chunk_kb} KiB n {n} kind {kind}")


# ---- b. every [h|d] pointer of the stage API -----------------------------------------------------

_STAGE = {}


def _dragon():
    if "dragon" not in _STAGE:
        Xf, Xm = load_pair("dragon")
        rng = np.random.default_rng(5)
        nrm = rng.normal(size=(Xm.shape[0], 3))
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        pl = rng.uniform(0, 1, Xm.shape[0])
        pl[::17] = np.nan  # "not estimated"
        mov_attr = [a.astype(np.float32) for a in (nrm[:, 0], nrm[:, 1], nrm[:, 2], pl)]
        _STAGE["dragon"] = (np.ascontiguousarray(Xf), np.ascontiguousarray(Xm), mov_attr)
    return _STAGE["dragon"]


def _stage_calls(e, kind, K):
    """The stage API on dragon with every [h|d] pointer in `kind`; returns every output."""
    lib, h = e._lib, e._h
    Xf, Xm, mov_attr = _dragon()
    nf, nm = Xf.shape[0], Xm.shape[0]
    sel = pointcloud.subsample_indices(nf, K).astype(np.int64)
    H = synthetic.H_from_rbp((0.01, -0.02, 0.015, 0.003, -0.002, 0.001))
    r = float(np.median(cKDTree(Xm).query(Xf[sel])[0]))  # keeps about half of the selection
    out = {}
    e.set_clouds(Xf, Xm)
    e.set_option("keep_knn", 1)
    # inputs
    sel_in = Buf(kind, K, np.int64).put(sel)  # a name keeps every buffer alive through its call
    e._check(lib.sicp_set_selected(h, sel_in.addr, K))
    n = C.c_int64(0)
    keep = Buf(kind, K, np.uint8)
    e._check(lib.sicp_select_in_range(h, _capi._d16(np.eye(4)), r, keep.addr, C.byref(n)))
    out["select_in_range keep"], out["select_in_range n_kept"] = keep.get(), np.int64(n.value)
    nrm = [Buf(kind, K, np.float32) for _ in range(4)]
    e._check(lib.sicp_estimate_normals(h, 10, *[b.addr for b in nrm]))
    for j, b in enumerate(nrm):
        out[f"estimate_normals {j}"] = b.get()
    kidx, kd2 = Buf(kind, (K, 10), np.int64), Buf(kind, (K, 10), np.float64)
    e._check(lib.sicp_get_knn(h, kidx.addr, kd2.addr))
    out["get_knn idx"], out["get_knn dist2"] = kidx.get(), kd2.get()
    # the normals back in with their signs flipped, so that the stored normals change
    given = [-out["estimate_normals 0"], -out["estimate_normals 1"], -out["estimate_normals 2"], out["estimate_normals 3"]]
    bufs = [Buf(kind, K, np.float32).put(a) for a in given]
    e._check(lib.sicp_set_normals(h, *[b.addr for b in bufs]))
    bufs = [Buf(kind, nm, np.float32).put(a) for a in mov_attr]
    e._check(lib.sicp_set_mov_normals(h, *[b.addr for b in bufs], float(np.deg2rad(80.0))))
    # outputs
    idx, dist = Buf(kind, K, np.int64), Buf(kind, K, np.float64)
    e._check(lib.sicp_match(h, _capi._d16(H), idx.addr, dist.addr))
    out["match idx"], out["match dist"] = idx.get(), dist.get()
    keep = Buf(kind, K, np.uint8)
    stats = (C.c_double * 4)()
    e._check(lib.sicp_reject(h, 0.3, keep.addr, C.byref(n), stats))
    n_kept = int(n.value)
    out["reject keep"], out["reject n_kept"], out["reject stats"] = keep.get(), np.int64(n_kept), np.array(stats)
    lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
    x, Hs, st, w = (C.c_double * 6)(), (C.c_double * 16)(), (C.c_double * 2)(), C.c_double(0)
    res = Buf(kind, n_kept, np.float64)
    e._check(lib.sicp_solve(h, C.byref(lsq), x, Hs, res.addr, st, C.byref(w)))
    out["solve residuals"], out["solve x"], out["solve H"] = res.get(), np.array(x), np.array(Hs)
    out["solve stats"], out["solve weight"] = np.array(st), np.float64(w.value)
    res = Buf(kind, n_kept, np.float64)
    e._check(lib.sicp_get_residuals(h, res.addr, n_kept, C.byref(n)))
    out["get_residuals"], out["get_residuals n"] = res.get(), np.int64(n.value)
    Xt = Buf(kind, (nm, 3), np.float64)
    e._check(lib.sicp_transform(h, _capi._d16(np.array(Hs).reshape(4, 4)), Xt.addr))
    out["transform"] = Xt.get()
    m = K // 3 + 1
    sel_out = Buf(kind, m, np.int64)
    e._check(lib.sicp_select_n_points(h, m, sel_out.addr))
    out["select_n_points"] = sel_out.get()
    return out


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K", [1000, 6000])  # one block, and the cooperative kernel (K > 4096)
def test_stage_api_pointers(eng, K, kind):
    key = ("stage", K)
    if key not in _STAGE:
        _options(eng, threads=0)
        _STAGE[key] = _stage_calls(eng, "P", K)
    base = _STAGE[key]
    assert 6 <= base["reject n_kept"] < K and 0 < base["select_in_range n_kept"] < K
    _options(eng)
    _same_all(_stage_calls(eng, kind, K), base, f"K {K} kind {kind}")


# ---- c. whole registrations ----------------------------------------------------------------------

_C3 = {}


def _c3():
    if "pair" not in _C3:
        Xf, Xm, _ = synthetic.c3_pair(1_000_000)
        _C3["pair"] = (Xf, Xm)
    return _C3["pair"]


def _result(r) -> dict:
    d = {"H": r.H, "X_t": _host(r.X_mov_transformed), "residuals": r.residuals,
         "iterations": np.int64(r.iterations), "converged": np.bool_(r.converged),
         "idx_selected": np.asarray(r.idx_selected),
         "x": np.array(r.rbp.get_parameter_attributes_as_list("estimated_value")),
         "sigma": np.array(r.rbp.get_parameter_attributes_as_list("estimated_uncertainty"))}
    for i, rec in enumerate(r.records):
        for k, v in rec.items():
            d[f"record {i} {k}"] = np.asarray(v)
    if r.normals is not None:
        for j, a in enumerate(r.normals):
            d[f"normals {j}"] = np.asarray(a)
    return d


REGISTER_CONFIGS = {"plain": {}, "overlap": dict(max_overlap_distance=1.0), "mov_neighbors": dict(mov_neighbors=10)}
OUT_KINDS = (None, "P", "H", "D", "D+")


@pytest.mark.parametrize("config", list(REGISTER_CONFIGS))
@pytest.mark.parametrize("staged", [False, True], ids=["fused", "staged"])
def test_register_every_kind(eng, staged, config):
    """sb.register on the C3 pair (1M <-> 1M, K = 100 000), one library call (fused) or stage by
    stage (want_normals=True); the overlap filter reverses the fused call's upload order."""
    Xf, Xm = _c3()
    kw = dict(REGISTER_CONFIGS[config], correspondences=100_000, want_normals=staged, engine=eng)
    base = {}
    for kind in CLOUD_KINDS:
        fix, Vf = _cloud(kind, Xf)
        mov, Vm = _cloud(kind, Xm)
        key = kind == "D32"
        if key not in base:
            _options(eng, threads=0)
            base[key] = _result(sb.register(Vf.copy(), Vm.copy(), **kw))
            _options(eng)
        for ok in OUT_KINDS:
            out = None if ok is None else Buf(ok, Xm.shape, np.float64)
            r = sb.register(fix, mov, transform_out=None if out is None else out.obj, **kw)
            got = _result(r)
            if out is not None:
                assert r.X_mov_transformed is out.obj
                got["X_t"] = out.get()
            _same_all(got, base[key], f"{'staged' if staged else 'fused'} {config} inputs {kind} transform_out {ok}")


def test_simpleicp_on_cuda_tensors(eng):
    Xf, Xm = _c3()
    _options(eng, threads=0)
    H0, X0, rbp0, res0 = sb.simpleicp(Xf, Xm, correspondences=100_000, engine=eng)
    _options(eng)
    H1, X1, rbp1, res1 = sb.simpleicp(torch.from_numpy(Xf).cuda(), torch.from_numpy(Xm).cuda(),
                                      correspondences=100_000, engine=eng)
    _same(H1, H0, "H")
    _same(_host(X1), _host(X0), "X_mov_transformed")
    _same(res1, res0, "residuals")
    for a in ("estimated_value", "estimated_uncertainty"):
        _same(np.array(rbp1.get_parameter_attributes_as_list(a)), np.array(rbp0.get_parameter_attributes_as_list(a)), a)


def _pair_table(res) -> dict:
    d = {"n_selected": np.asarray(res.n_selected)}
    for i, p in enumerate(res):
        for f, _ in _capi.PairResult._fields_:
            d[f"pair {i} {f}"] = np.array(getattr(p, f))
    return d


@pytest.mark.parametrize("opts", [dict(), dict(max_overlap_distance=1.0, mov_neighbors=10)], ids=["plain", "filter_mov"])
def test_register_batch_mixed_kinds(eng, opts):
    """8 C5 pairs; pair i takes its fixed cloud in kind i and its movable cloud in kind i + 3."""
    raw = [synthetic.c5_pair(i)[:2] for i in range(8)]
    pairs, values = [], []
    for i, (Xf, Xm) in enumerate(raw):
        f, Vf = _cloud(CLOUD_KINDS[i % 8], Xf)
        m, Vm = _cloud(CLOUD_KINDS[(i + 3) % 8], Xm)
        pairs.append((f, m))
        values.append((Vf, Vm))
    params = eng.run_params(0.3, 1.0, 100, eng.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
    _options(eng, threads=0)
    base = _pair_table(eng.register_batch(values, 1000, 10, params, **opts))
    _options(eng)
    assert all(base[f"pair {i} status"] == 0 for i in range(8))
    _same_all(_pair_table(eng.register_batch(pairs, 1000, 10, params, **opts)), base, f"batch {opts}")


@pytest.mark.parametrize("opts", [dict(), dict(max_overlap_distance=1.0, mov_neighbors=10)], ids=["plain", "filter_mov"])
def test_register_pairs_movable_only_kinds(eng, opts):
    """register_pairs on 8 C5 pairs and one more: pair i (i < 8) is (fixed cloud i, movable cloud
    8 + i), the movable cloud in kind i, so the movable-only clouds, which cross PCIe on the copy
    stream, take every kind; pair 8 is (fixed cloud 1, fixed cloud 0), so cloud 0 is in both roles
    and clouds 1-7 are fixed only.  The fixed clouds are pageable."""
    raw = [synthetic.c5_pair(i)[:2] for i in range(8)]
    clouds, values = [Xf for Xf, _ in raw], [Xf for Xf, _ in raw]
    for i, (_, Xm) in enumerate(raw):
        m, Vm = _cloud(CLOUD_KINDS[i], Xm)
        clouds.append(m)
        values.append(Vm)
    edges = [(i, 8 + i) for i in range(8)] + [(1, 0)]
    params = eng.run_params(0.3, 1.0, 100, eng.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
    _options(eng, threads=0)
    base = _pair_table(eng.register_pairs([V.copy() for V in values], edges, 1000, 10, params, **opts))
    _options(eng)
    assert all(base[f"pair {i} status"] == 0 for i in range(len(edges)))
    _same_all(_pair_table(eng.register_pairs(clouds, edges, 1000, 10, params, **opts)), base, f"pairs {opts}")


_MAP = {}


def _map_data():
    """A 2M-point surface map (48 MB: the threaded staging) and 4 tiles of a second realisation,
    each moved by a small rigid transform, with their priors in radians."""
    if "map" not in _MAP:
        X = synthetic.surface(2_000_000, 80_000, extent=120.0)
        second = synthetic.surface(2_000_000, 80_001, extent=120.0)
        rng = np.random.default_rng(80_000)
        scans, rows = [], []
        for x0, y0, w in ((10, 10, 25), (60, 40, 30), (90, 85, 28), (30, 70, 20)):
            m = (second[:, 0] >= x0) & (second[:, 0] < x0 + w) & (second[:, 1] >= y0) & (second[:, 1] < y0 + w)
            true = np.concatenate((np.deg2rad(rng.uniform(-1, 1, 3)), rng.uniform(-0.3, 0.3, 3)))
            scans.append(np.ascontiguousarray(synthetic.apply_H(second[m], np.linalg.inv(synthetic.H_from_rbp(true)))))
            rows.append(true + np.concatenate((rng.normal(0, 0.001, 3), rng.normal(0, 0.02, 3))))
        _MAP["map"] = (X, scans, np.array(rows))
    return _MAP["map"]


def _map_run(e, X_map, scans, rows):
    e.set_map(X_map)
    params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
    return _pair_table(e.register_to_map(scans, 1000, 10, params, max_overlap_distance=1.0, observed=rows))


def _map_base(e):
    if "base" not in _MAP:
        X, scans, rows = _map_data()
        _options(e, threads=0)
        _MAP["base"] = _map_run(e, X.copy(), scans, rows)
        assert all(_MAP["base"][f"pair {i} status"] == 0 for i in range(len(scans)))
    return _MAP["base"]


@pytest.mark.parametrize("chunk_kb", [64, 100, 2048, 4096])
@pytest.mark.parametrize("threads", [0, 1, 2, 3, 8])
def test_map_from_pageable(eng, threads, chunk_kb):
    base = _map_base(eng)
    X, scans, rows = _map_data()
    for kind in ("P", "P+"):
        _options(eng, threads, chunk_kb)
        _same_all(_map_run(eng, _cloud(kind, X)[0], scans, rows), base, f"map {kind} threads {threads} chunk {chunk_kb}")


@pytest.mark.parametrize("kind", [k for k in CLOUD_KINDS if k not in ("P", "P+", "D32")])
def test_map_from_every_kind(eng, kind):
    """The map from pinned, device, offset device, CPU tensor and non-contiguous sources; the
    scans in rotating exact kinds."""
    base = _map_base(eng)
    X, scans, rows = _map_data()
    _options(eng)
    scans_k = [_cloud(KINDS[(j + CLOUD_KINDS.index(kind)) % 5], S)[0] for j, S in enumerate(scans)]
    _same_all(_map_run(eng, _cloud(kind, X)[0], scans_k, rows), base, f"map {kind}")


# ---- d. the transform against exact arithmetic ---------------------------------------------------

def _round(q: Fraction) -> float:
    return q.numerator / q.denominator  # int / int is correctly rounded (to nearest, ties to even)


def _emulate(H, X):
    """k_transform's expression per output coordinate i, fma(r_i2, z, fma(r_i1, y, r_i0 x)) + t_i,
    with every operation rounded once (float(Fraction) rounds correctly; Python 3.12 has no
    math.fma), and the exact rational value of (R p + t)_i with M_i = sum_j |r_ij p_j|."""
    R = [[Fraction(float(H[i, j])) for j in range(3)] for i in range(3)]
    t = [Fraction(float(H[i, 3])) for i in range(3)]
    out, exact, mag = np.empty(X.shape), [], []
    for k, row in enumerate(X):
        p = [Fraction(float(v)) for v in row]
        ex_row, mag_row = [], []
        for i in range(3):
            a = _round(R[i][0] * p[0])
            b = _round(R[i][1] * p[1] + Fraction(a))
            c = _round(R[i][2] * p[2] + Fraction(b))
            out[k, i] = _round(Fraction(c) + t[i])
            ex_row.append(R[i][0] * p[0] + R[i][1] * p[1] + R[i][2] * p[2] + t[i])
            mag_row.append(abs(R[i][0] * p[0]) + abs(R[i][1] * p[1]) + abs(R[i][2] * p[2]))
        exact.append(ex_row)
        mag.append(mag_row)
    return out, exact, mag


# Error bound of that expression, u = 2^-53 (round to nearest), a, b, c the three products, E the
# exact result, M = |a| + |b| + |c|:
#   |fl(a) - a| <= u|a|
#   |q - (a + b)| <= u|b + fl(a)| + u|a| <= u(2|a| + |b|) + u^2 |a|          q = fl(b + fl(a))
#   |s - (a + b + c)| <= u|c + q| + |q - (a + b)| <= u(3|a| + 2|b| + |c|) + O(u^2 M) <= 3uM (1 + 2u)
#   |fl(s + t) - E| <= u|s + t| + |s - (a+b+c)| <= u|E| + 3uM (1 + 2u)^2
# i.e. a few ulps of the largest term.  The bound checked: u (|E| + 3M) (1 + 2^-48).
def _check_bound(Y, exact, mag, what):
    u = Fraction(1, 2**53)
    for k in range(Y.shape[0]):
        for i in range(3):
            err = abs(Fraction(float(Y[k, i])) - exact[k][i])
            bound = u * (abs(exact[k][i]) + 3 * mag[k][i]) * (1 + Fraction(1, 2**48))
            assert err <= bound, f"{what}: row {k} coordinate {i}: error {float(err):.3e} > bound {float(bound):.3e}"


ORIGINS = {"origin": np.zeros(3), "utm": np.array([612_345.0, 5_432_109.0, 250.0])}
TRANSFORM_N = (1, 2, 3, 511, 512, 513, 4097, 1_000_000)


@pytest.mark.parametrize("n", TRANSFORM_N)
@pytest.mark.parametrize("origin", list(ORIGINS))
def test_transform_rounds_like_its_expression(eng, origin, n):
    """Odd n exercise the tail thread, 511 / 512 / 513 and 4097 the 256-thread block edges."""
    rng = np.random.default_rng(_seed("transform", origin, n))
    X = ORIGINS[origin] + rng.uniform(-500.0, 500.0, (n, 3))
    H = synthetic.H_from_rbp((0.3, -1.1, 2.4, 12.5, -7.25, 3.0))  # a general rotation
    if n > 20_000:
        rows = np.unique(np.concatenate((np.arange(1000), np.arange(n - 1000, n),
                                         rng.choice(n, 20_000, replace=False))))
    else:
        rows = np.arange(n)
    want, exact, mag = _emulate(H, X[rows])
    _check_bound(want, exact, mag, f"{origin} n {n} emulation")
    _options(eng)
    eng.set_clouds(X[:1], X)
    for kind in KINDS:
        out = Buf(kind, (n, 3), np.float64)
        assert eng.transform(H, out=out.obj) is out.obj
        _same(out.get()[rows], want, f"{origin} n {n} out {kind}")


# ---- e. recovery after an abandoned upload -------------------------------------------------------

def test_abandoned_upload_then_every_source(eng):
    """sicp_set_clouds starts the fixed cloud's threaded upload in the background, then builds the
    movable grid, which refuses a NaN.  The call must return only when no transfer of the
    abandoned job is still running: the next upload into the same device buffer may come from
    another stream (a device source, or a pageable one on fewer workers).  The race that a
    missing wait opens cannot be forced from here; what this pins is the contract that the same
    engine afterwards uploads every byte from any source."""
    n = 1_000_000
    for threads, kind, next_threads in ((2, "D", None), (8, "P", 1)):
        _options(eng, threads)
        rng = np.random.default_rng(_seed("abandon", threads))
        X_fix = rng.normal(size=(n, 3)) * 50.0
        X_mov = X_fix[: n // 2].copy()
        X_mov[n // 4, 1] = np.nan
        with pytest.raises(_capi.SicpError) as err:
            eng.set_clouds(X_fix, X_mov)
        assert err.value.code == _capi.SICP_ERR_BAD_ARG, err.value
        if next_threads is not None:
            eng.set_option("upload_threads", next_threads)
        X = np.random.default_rng(_seed("abandon probe", threads)).normal(size=(n, 3)) * 50.0
        _probe(eng, kind, X, f"after an abandoned upload on {threads} workers: {kind}")


# ---- f. an output on another GPU -----------------------------------------------------------------

def test_transform_out_on_another_gpu(eng):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    Xf, Xm, _ = synthetic.c5_pair(0)
    _options(eng, threads=0)
    base = _result(sb.register(Xf, Xm, engine=eng, want_normals=False))
    eng.set_clouds(Xf, Xm)
    H = synthetic.H_from_rbp((0.3, -1.1, 2.4, 12.5, -7.25, 3.0))
    want = _host(eng.transform(H))
    _options(eng)
    m = 3 * Xm.shape[0]
    for off in (0, 1):  # aligned, and one element off
        buf = torch.full((m + 2,), np.nan, dtype=torch.float64, device="cuda:1")
        out = buf[off:off + m].view(-1, 3)
        got = _result(sb.register(Xf, Xm, engine=eng, want_normals=False, transform_out=out))
        got["X_t"] = _host(out)
        _same_all(got, base, f"transform_out on cuda:1 offset {off}")
        eng.set_clouds(Xf, Xm)
        out.fill_(np.nan)
        _same(_host(eng.transform(H, out=out)), want, f"transform out= on cuda:1 offset {off}")
        assert torch.isnan(buf[:off]).all() and torch.isnan(buf[off + m:]).all(), "guard overwritten"
