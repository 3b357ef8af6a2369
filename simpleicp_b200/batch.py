"""Batched registration of independent (X_fix, X_mov) pairs, sharded over GPUs.

Independent pairs share nothing (SURVEY.md §8e): each rank registers its static share on its
own GPU with the single-GPU pipeline and the only exchange is one all-gather of a fixed-size
record per pair — H (16 f64), iterations, kept correspondences, mean and std of the final
residuals — over NCCL (gloo on CPU-only hosts for the tests of the sharding logic).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

RECORD_LEN = 20  # H (16) + iterations + n_kept + mean + std


def shard_pairs(n_pairs: int, world_size: int, rank: int) -> List[int]:
    """Static round-robin assignment: pair i belongs to rank i % world_size."""
    if world_size < 1 or not 0 <= rank < world_size:
        raise ValueError("invalid rank / world_size")
    return list(range(rank, n_pairs, world_size))


def pack_record(H: np.ndarray, iterations: int, n_kept: int, mean: float, std: float) -> np.ndarray:
    r = np.empty(RECORD_LEN)
    r[:16] = np.asarray(H, dtype=float).reshape(16)
    r[16:] = (iterations, n_kept, mean, std)
    return r


def _failed_record(code: int) -> np.ndarray:
    """The record of a pair that could not be registered: NaN, iterations = -code."""
    return pack_record(np.full((4, 4), np.nan), -int(code), 0, np.nan, np.nan)


def _pair_record(r, kind: str, number: int, messages: List[str]) -> np.ndarray:
    """The record of PairResult `r`, pair or edge `number` of the call; for one that failed the
    library's status also goes to `messages`."""
    if r.status == 0:
        return pack_record(np.array(r.H).reshape(4, 4), r.iterations, r.n_kept, r.mean_res, r.std_res)
    messages.append(f"{kind} {number}: library status {r.status}")
    return _failed_record(r.status)


def _raise_failed(table: np.ndarray, on_error: str, messages: List[str], results=None) -> None:
    """BatchError when rows of `table` failed (iterations < 0) and `on_error` is "raise"."""
    failed = np.flatnonzero(table[:, 16] < 0)
    if failed.size and on_error == "raise":
        raise BatchError(table, failed, messages, results)


def gather_records(local: np.ndarray, n_pairs: int, world_size: int, rank: int, dist=None,
                   device=None) -> np.ndarray:
    """All-gather the per-pair records.  `local` is (len(shard), RECORD_LEN) in shard order;
    returns (n_pairs, RECORD_LEN) in pair order on every rank."""
    if world_size == 1 or dist is None:
        out = np.zeros((n_pairs, RECORD_LEN))
        out[shard_pairs(n_pairs, 1, 0)] = local
        return out
    import torch

    per = (n_pairs + world_size - 1) // world_size  # equal-size slots, last ones may be padding
    buf = torch.full((per, RECORD_LEN), float("nan"), dtype=torch.float64, device=device)
    if local.shape[0]:
        buf[: local.shape[0]] = torch.from_numpy(np.ascontiguousarray(local)).to(buf.device)
    gathered = torch.empty((world_size * per, RECORD_LEN), dtype=torch.float64, device=device)
    dist.all_gather_into_tensor(gathered, buf)
    g = gathered.cpu().numpy().reshape(world_size, per, RECORD_LEN)
    out = np.zeros((n_pairs, RECORD_LEN))
    for r in range(world_size):
        ids = shard_pairs(n_pairs, world_size, r)
        out[ids] = g[r, : len(ids)]
    return out


def tile_slabs(X_fix: np.ndarray, X_mov: np.ndarray, n_slabs: int, overlap: float, axis: int = 0):
    """Cut a large pair into `n_slabs` overlapping slabs along `axis` (BASELINE.json configs[3],
    SURVEY.md section 8d C4): equal-count quantile cuts of the fixed cloud's coordinate, the same
    cuts for both clouds, every slab widened by `overlap` on both sides.  Each slab is an
    independent registration.  Returns a list of (X_fix_slab, X_mov_slab)."""
    if n_slabs < 1:
        raise ValueError("n_slabs must be >= 1")
    cuts = np.quantile(X_fix[:, axis], np.linspace(0.0, 1.0, n_slabs + 1))
    cuts[0], cuts[-1] = -np.inf, np.inf
    out = []
    for s in range(n_slabs):
        lo, hi = cuts[s] - overlap, cuts[s + 1] + overlap
        mf = (X_fix[:, axis] >= lo) & (X_fix[:, axis] < hi)
        mm = (X_mov[:, axis] >= lo) & (X_mov[:, axis] < hi)
        out.append((np.ascontiguousarray(X_fix[mf]), np.ascontiguousarray(X_mov[mm])))
    return out


# Engines (one CUDA stream + one libsicp_b200 context each) are kept between calls: creating a
# context and growing its device buffers costs far more than one small registration.
_ENGINES: dict = {}


def _engine_pool(device: int, n: int):
    import torch

    from . import _capi

    pool = _ENGINES.setdefault(int(device), [])
    with torch.cuda.device(device):
        while len(pool) < n:
            stream = torch.cuda.Stream(device=device)
            pool.append((stream, _capi.Engine(device, stream=int(stream.cuda_stream))))
    return pool


def close_engine_pool() -> None:
    """Release the engines simpleicp_batch keeps between calls."""
    for pool in _ENGINES.values():
        for _, eng in pool:
            eng.close()
    _ENGINES.clear()
    for eng in _BATCH_ENGINES.values():
        eng.close()
    _BATCH_ENGINES.clear()


def simpleicp_batch(
    pairs: Sequence[Tuple[np.ndarray, np.ndarray]] | Callable[[int], Tuple[np.ndarray, np.ndarray]],
    n_pairs: Optional[int] = None,
    *,
    rank: int = 0,
    world_size: int = 1,
    dist=None,
    device: int = 0,
    register_fn=None,
    concurrency: int = 4,
    on_error: str = "raise",
    batch_size: int = 64,
    engine: str = "batched",
    full_output: bool = False,
    **run_kwargs,
):
    """Register every pair; returns the (n_pairs, 20) record table on every rank.

    `pairs` is a sequence or a generator function i -> (X_fix, X_mov) (so that ranks only
    materialise their own share).  `register_fn` defaults to the GPU pipeline
    (simpleicp_b200.register on cuda:`device`); tests inject a stub to exercise the sharding and
    the collective on CPU.  On the GPU path `concurrency` engines, each on its own CUDA stream and
    driven by its own thread (the C calls release the GIL), work through the rank's share so the
    host round trips of small registrations overlap.

    `engine="batched"` (default) hands the rank's share to the library's batched engine in chunks
    of `batch_size` pairs (sicp_register_batch: one set of kernel launches per stage and per
    iteration for the whole chunk, a block per pair for reject + solve, per-pair stop flags);
    pairs it does not cover (more than 4096 correspondences, debug output) and `engine="pool"`
    use the concurrent per-pair engines described above.

    `rbp_observed_values` is either the common 6-tuple or an array of shape (n_pairs, 6) indexed
    by pair number, one prior per pair (e.g. a GNSS/INS or odometry pose; angles in degrees):
    each pair starts from its own row, which is also the transform its overlap filter runs under.
    Every row is checked before any registration starts.

    `mov_neighbors=k` estimates every movable cloud's normals from k neighbours (as
    `pc_mov.estimate_normals(k)` would) and rejects correspondences by the movable planarity too;
    `max_angle_between_normals` (degrees, needs `mov_neighbors`) also by the angle between the
    normals.  Both are checked before any registration starts and are served by the batched engine.

    A pair that cannot be registered (no overlap, fewer than 6 correspondences: ordinary
    data-dependent outcomes) gets a NaN record whose `iterations` field is minus the library's
    status code; every rank still takes part in the collective.  Afterwards `on_error="raise"`
    raises BatchError (same on every rank, `.table` holds the full table, `.failed` the pair
    numbers), `on_error="nan"` just returns the table.

    `full_output=True` returns `(table, results)` instead, with the same table.  `results[i]` is
    what `register` returns for pair i -- `H`, `X_mov_transformed`, `rbp` with the estimated
    uncertainties, `residuals`, `records`, `iterations`, `converged`; fields the batched engine
    has no equivalent for are None -- and None for a pair that failed or belongs to another rank
    (only the table is exchanged between ranks).  Pairs served per pair (`engine="pool"`, more
    than 4096 correspondences, `register_fn`) give the objects `register` / `register_fn`
    returned.  BatchError then carries `.results` too.
    """
    if n_pairs is None:
        n_pairs = len(pairs)  # type: ignore[arg-type]
    get = pairs if callable(pairs) else (lambda i: pairs[i])  # type: ignore[index]
    mine = shard_pairs(n_pairs, world_size, rank)
    local = np.zeros((len(mine), RECORD_LEN))
    found: List = [None] * len(mine)  # full_output: the result object of each pair of the share
    rows = _per_pair_observed(run_kwargs, n_pairs)
    _check_mov_kwargs(run_kwargs)

    def kw_of(i):
        return run_kwargs if rows is None else {**run_kwargs, "rbp_observed_values": rows[i]}

    def record(res):
        last = res.records[res.iterations - 1]
        return pack_record(res.H, res.iterations, last["n_kept"], last["mean_res"], last["std_res"])

    def guarded(fn, j, Xf, Xm, **kw):
        try:
            res = fn(Xf, Xm, **kw)
            if full_output:
                found[j] = res
            return record(res)
        except Exception as e:  # noqa: BLE001 — recorded per pair, reported after the gather
            code = getattr(getattr(e, "__cause__", None) or e, "code", None)
            msg = str(e)
            if code is None:
                code = 2 if "overlap" in msg else (3 if "correspondences" in msg else 99)
            messages.append(msg)
            return _failed_record(code)

    messages: List[str] = []
    if register_fn is not None:
        for j, i in enumerate(mine):
            Xf, Xm = get(i)
            local[j] = guarded(register_fn, j, Xf, Xm, **kw_of(i))
    elif engine == "batched" and _batchable(run_kwargs):
        # results= only when asked for: the default call is unchanged
        _run_batched(get, mine, local, device, batch_size, run_kwargs, messages, rows,
                     **({"results": found} if full_output else {}))
    else:
        import threading

        import torch

        from .simpleicp import register

        run_kwargs.setdefault("want_normals", False)  # one fused sicp_register call per pair
        n_workers = max(1, min(concurrency, len(mine)))
        errors = []
        pool = _engine_pool(device, n_workers)
        todo, lock = iter(range(len(mine))), threading.Lock()

        def worker(w):
            try:
                with torch.cuda.device(device):
                    _, eng = pool[w]
                    while True:
                        with lock:  # dynamic hand-out: iteration counts (3 .. max_iterations) vary a lot
                            j = next(todo, None)
                        if j is None:
                            break
                        Xf, Xm = get(mine[j])
                        local[j] = guarded(register, j, Xf, Xm, engine=eng, **kw_of(mine[j]))
            except Exception as e:  # surfaced after the join
                errors.append(e)

        threads = [threading.Thread(target=worker, args=(w,)) for w in range(n_workers)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:  # not a per-pair outcome (bad generator, lost device): NaN for what is missing
            messages.append(repr(errors[0]))
            done = np.isfinite(local[:, 16]) & (local[:, 16] != 0)
            local[~done] = _failed_record(99)
    return _gather_share(local, found, mine, n_pairs, rank, world_size, dist, device, on_error, full_output, messages)


def _gather_share(local, found, mine, n_pairs, rank, world_size, dist, device, on_error, full_output, messages):
    """The end of simpleicp_batch and simpleicp_edges: the rank's records `local` (and with
    full_output its result objects `found`, both in the order of its share `mine`) all-gathered
    into the table, BatchError per `on_error`, the return value."""
    dev = None
    if dist is not None and world_size > 1:
        import torch

        dev = torch.device("cuda", device) if dist.get_backend() == "nccl" else torch.device("cpu")
    table = gather_records(local, n_pairs, world_size, rank, dist, dev)
    results = None
    if full_output:
        results = [None] * n_pairs
        for j, i in enumerate(mine):
            results[i] = found[j]
    _raise_failed(table, on_error, messages, results)
    return (table, results) if full_output else table


def simpleicp_edges(clouds: Sequence, edges, *, rank: int = 0, world_size: int = 1, dist=None, device: int = 0,
                    batch_size: int = 64, on_error: str = "raise", full_output: bool = False, **run_kwargs):
    """Register many pairs drawn from one set of clouds; returns simpleicp_batch's (n_edges, 20)
    record table on every rank.

    `clouds` is a sequence of (n_i, 3) NumPy arrays or CUDA tensors; `edges` is (n_edges, 2) of
    integer (fixed, movable) indices into it, e.g. the edges (i, i + 1) and (i, i + 2) of a scan
    sequence, loop-closure candidates, or one pair repeated under several priors.  Edge i's row
    equals that of ``simpleicp_batch([(clouds[a], clouds[b]) for a, b in edges], ...)`` bit for
    bit, but every cloud a library call uses is uploaded and gridded once per call, and with
    `mov_neighbors` given its normals once, however many edges share it (sicp_register_pairs).

    Edges are taken in order, `batch_size` per library call; each call passes only the clouds its
    edges reference (edge_chunks).  Edge i belongs to rank i % world_size, and only the table is
    exchanged.  ``rbp_observed_values`` is the common 6-tuple or one row per edge (degrees), each
    edge's prior.  The run() arguments served are those of the batched engine without
    ``want_normals`` (at most 4096 correspondences); anything else is a TypeError.  `on_error`,
    `full_output` and BatchError are as in simpleicp_batch."""
    _check_run_keys(run_kwargs, _EDGE_KEYS, "simpleicp_edges", "edge")
    e = _check_edges(edges, len(clouds))
    n = e.shape[0]
    rows = _per_pair_observed(run_kwargs, n)
    _check_mov_kwargs(run_kwargs)
    mine = shard_pairs(n, world_size, rank)
    local = np.zeros((len(mine), RECORD_LEN))
    found: List = [None] * len(mine)
    messages: List[str] = []
    _run_batched(lambda i: clouds[i], mine, local, device, batch_size, run_kwargs, messages, rows, edges=e,
                 **({"results": found} if full_output else {}))
    return _gather_share(local, found, mine, n, rank, world_size, dist, device, on_error, full_output, messages)


# simpleicp_joint's solvers and the free clouds each takes (option joint_solver 0 and 1)
_JOINT_SOLVERS = {"dense": 256, "sparse": 16384}

# run() arguments simpleicp_joint serves (sicp_register_joint, always the linearised rules)
_JOINT_KEYS = {"correspondences", "neighbors", "min_planarity", "min_change", "max_iterations", "max_overlap_distance"}


class JointResult:
    """simpleicp_joint's return value: H (n_clouds, 4, 4) final poses, world <- cloud; table the
    (n_edges, 20) record table of simpleicp_edges with H = the final T_a^-1 T_b of each edge;
    iterations and converged of the call; results (full_output) the per-edge result objects; with
    covariances=True or "selected" cov (n_clouds, 6, 6), edge_cov (n_edges, 6, 6) and s0, the
    a-posteriori covariances of sicp_get_joint_covariances (else None); with relative observations
    relative_misclosure (n_rel, 6), each observation's (rotvec(R_Z R_ab^T), t_Z - t_ab) at the
    returned poses (else None)."""

    def __init__(self, H, table, iterations, converged, results=None, cov=None, edge_cov=None, s0=None,
                 relative_misclosure=None):
        self.H, self.table, self.iterations, self.converged, self.results = H, table, iterations, converged, results
        self.cov, self.edge_cov, self.s0 = cov, edge_cov, s0
        self.relative_misclosure = relative_misclosure


def simpleicp_joint(clouds: Sequence, edges, *, fixed=(0,), H0=None, device: int = 0, on_error: str = "raise",
                    full_output: bool = False, covariances=False, solver: str = "dense",
                    prior_poses=None, prior_weights=None, relative_pairs=None, relative_poses=None,
                    relative_weights=None, **run_kwargs) -> JointResult:
    """Register many clouds jointly (multi-scan ICP): one pose per cloud such that every edge
    (a, b) of `edges` -- scan-to-scan pairs such as (i, i + 1), (i, i + 2) and loop closures -- is
    registered consistently.  Each iteration matches every edge as simpleicp_edges would under the
    linearised rules (median / MAD of all distances, sigma = 1.4826 MAD, point-to-plane rows of the
    C++ driver) and solves ONE least-squares problem for the increments of all free clouds; the
    clouds listed in `fixed` (indices, at least one unless pose priors anchor every component) hold
    their pose.  `H0` (n_clouds, 4, 4) are the start poses (None: identity), world <- cloud.

    The run() arguments served are correspondences (<= 4096), neighbors, min_planarity,
    min_change, max_iterations and max_overlap_distance; anything else is a TypeError.  Every free
    cloud an edge references must be connected to a fixed cloud through the edges, and there may be
    at most 256 of them (16 384 with solver="sparse").  A cloud no edge references may be None; it
    keeps its H0.  One library call on one device (sicp_register_joint).  `on_error` and
    `full_output` are as in simpleicp_edges: an edge that failed (no overlap, too few
    correspondences) has its status in the table and raises BatchError under "raise"; a failure of
    the whole call (SICP_ERR_SINGULAR, or a free cloud left without a path to a fixed one by the
    edges without overlap) raises SicpError.

    `covariances=True` also returns the a-posteriori covariances of the final iteration
    (sicp_get_joint_covariances, DESIGN.md §6.9): cov[c] of cloud c's (rotation increment, origin
    displacement) in the world frame, zeros for a fixed cloud and NaN for a cloud no edge
    references; edge_cov[e] of edge (a, b)'s (rotation increment, displacement of b's origin) in
    frame a; s0 the a-posteriori standard deviation of unit weight.  `covariances="selected"`
    returns the same under either solver (sicp_get_joint_selected_covariances, DESIGN.md §6.14):
    under "dense" the bits of True, under "sparse" the blocks by selected inversion of the sparse
    solve's factor.  True under "sparse" is a ValueError.

    `solver` picks the solve of the joint system (option joint_solver): "dense" (the default: the
    dense Cholesky of DESIGN.md §6.9, at most 256 free clouds, the only one with covariances=True) or
    "sparse" (a supernodal Cholesky over a nested-dissection ordering of the edge graph, DESIGN.md
    §6.11: the same system and rule, up to rounding, for up to 16 384 free clouds).

    `prior_poses` (n_clouds, 4, 4) and `prior_weights` (n_clouds, 6), given together, are weighted
    observations of each cloud's pose (DESIGN.md §6.12), e.g. GNSS/INS poses: cloud c's rotation
    and origin are pulled towards prior_poses[c] with the weights (w_wx, w_wy, w_wz, w_x, w_y, w_z)
    in world axes, 1/rad^2 and 1/m^2 relative to a point-to-plane row in metres, i.e.
    (sigma_row / sigma_prior)^2; 0 leaves a component unobserved.  Only the priors of free clouds
    with a non-zero weight are read (any other pose may be NaN); weights must be finite and >= 0
    and a read pose finite and rigid (to 1e-6).  A free cloud whose six weights are all > 0
    anchors its component of the edge graph as a fixed cloud does, so with priors `fixed` may be
    empty.  Both solvers take priors; covariances=True includes them.

    `relative_pairs` (n_rel, 2), `relative_poses` (n_rel, 4, 4) and `relative_weights` (n_rel, 6),
    given together, are weighted observations of the relative pose of two clouds (DESIGN.md
    §6.13), e.g. odometry between consecutive scans: observation k pulls T_a^-1 T_b of its clouds
    (a, b) towards relative_poses[k] (cloud b in frame a) with the weights (w_ax, w_ay, w_az, w_x,
    w_y, w_z) in frame-a axes, in the units of the prior weights.  Both clouds must be referenced
    by an edge.  Only observations with a non-zero weight and a free cloud are read (any other pose
    may be NaN); weights must be finite and >= 0 and a read pose finite and rigid (to 1e-6).  An
    observation whose six weights are all > 0 links its two clouds' components of the edge graph,
    e.g. across a stretch without overlap.  Both solvers take them; covariances=True includes them;
    the result's relative_misclosure shows how far each is from the returned poses."""
    selected = isinstance(covariances, str) and covariances == "selected"
    if not selected and not isinstance(covariances, (bool, np.bool_)):
        raise TypeError(f"covariances must be True, False or 'selected', got {covariances!r}")
    if not isinstance(solver, str) or solver not in _JOINT_SOLVERS:
        raise ValueError(f"solver must be 'dense' or 'sparse', got {solver!r}")
    if not selected and covariances and solver == "sparse":
        raise ValueError("covariances=True needs solver='dense': the sparse solve has no covariances; "
                         "covariances='selected' serves both solvers")
    _check_run_keys(run_kwargs, _JOINT_KEYS, "simpleicp_joint", "edge")
    n_clouds = len(clouds)
    e = _check_edges(edges, n_clouds)
    if e.shape[0] < 1:
        raise ValueError("simpleicp_joint needs at least one edge")
    if np.any(e[:, 0] == e[:, 1]):
        raise ValueError(f"edges must not be self edges: edge {int(np.flatnonzero(e[:, 0] == e[:, 1])[0])}")
    priors = prior_poses is not None or prior_weights is not None
    if priors and (prior_poses is None or prior_weights is None):
        raise ValueError("prior_poses and prior_weights must be given together")
    rel = relative_pairs is not None or relative_poses is not None or relative_weights is not None
    if rel and (relative_pairs is None or relative_poses is None or relative_weights is None):
        raise ValueError("relative_pairs, relative_poses and relative_weights must be given together")
    fx = np.asarray(fixed)
    if (priors or rel) and fx.size == 0:  # priors (linked by observations) may anchor every component
        fx = fx.astype(np.int64).reshape(0)
    if fx.ndim != 1 or (fx.size < 1 and not (priors or rel)) or not np.issubdtype(fx.dtype, np.integer):
        raise ValueError("fixed must be a sequence of at least one integer cloud index"
                         f"{' (or none, with priors)' if priors or rel else ''}")
    if fx.size and (fx.min() < 0 or fx.max() >= n_clouds):
        raise ValueError(f"fixed must index the {n_clouds} clouds")
    is_fixed = np.zeros(n_clouds, dtype=bool)
    is_fixed[fx] = True
    if H0 is not None:
        H0 = _finite_array(H0, "H0", (n_clouds, 4, 4))
    used = np.zeros(n_clouds, dtype=bool)
    used[e.ravel()] = True
    free = used & ~is_fixed
    cap = _JOINT_SOLVERS[solver]
    if not 1 <= int(free.sum()) <= cap:
        raise ValueError(f"the edges must reference between 1 and {cap} free clouds"
                         f"{' under solver=sparse' if solver == 'sparse' else ''}, got {int(free.sum())}")
    full = np.zeros(n_clouds, dtype=bool)
    if priors:
        prior_poses, prior_weights, full = _joint_priors(prior_poses, prior_weights, free)
    links = np.zeros((0, 2), dtype=np.int64)
    if rel:
        relative_pairs, relative_poses, relative_weights, link = _joint_relative(
            relative_pairs, relative_poses, relative_weights, used, free)
        links = relative_pairs[link]
    up = list(range(n_clouds))

    def root(i):
        while up[i] != i:
            up[i] = up[up[i]]
            i = up[i]
        return i

    for a, b in np.concatenate((e, links)):
        up[root(int(a))] = root(int(b))
    anchored = {root(i) for i in np.flatnonzero(is_fixed | full)}
    lost = [i for i in np.flatnonzero(free) if root(int(i)) not in anchored]
    if lost:
        raise ValueError(f"free cloud {int(lost[0])} has no path to a fixed cloud over the edges"
                         f"{' and the relative observations with six non-zero weights' if rel else ''}"
                         f"{' and no pose prior with six non-zero weights in its component' if priors else ''}")
    for i in np.flatnonzero(used):
        if clouds[i] is None:
            raise ValueError(f"cloud {int(i)} is referenced by an edge but is None")
    import torch

    with torch.cuda.device(device):
        eng = _batch_engine(device)
        lsq = eng.lsq_params((0.0,) * 6, (0.0,) * 6, [0.0] * 6, 1)
        params = eng.run_params(run_kwargs.get("min_planarity", 0.3), run_kwargs.get("min_change", 1.0),
                                run_kwargs.get("max_iterations", 100), lsq)
        mod = float(run_kwargs.get("max_overlap_distance", np.inf))
        # every call sets the option: the engine is shared by the calls on this device
        eng.set_option("joint_solver", 1 if solver == "sparse" else 0)
        H, res = eng.register_joint(list(clouds), e, is_fixed, H0, run_kwargs.get("correspondences", 1000),
                                    run_kwargs.get("neighbors", 10), params, mod if np.isfinite(mod) else -1.0,
                                    prior_poses, prior_weights, *((relative_pairs, relative_poses, relative_weights)
                                                                  if rel and len(relative_pairs) else ()))
        n = e.shape[0]
        table = np.zeros((n, RECORD_LEN))
        messages: List[str] = []
        for j, r in enumerate(res):
            table[j] = _pair_record(r, "edge", j, messages)
        results = None
        if full_output:
            results = [None if o is None else _batch_result(r, o, np.zeros(6), (0.0,) * 6)
                       for r, o in zip(res, eng.batch_outputs(res))]
        if selected:
            cov = eng.joint_selected_covariances(n_clouds, n)
        else:
            cov = eng.joint_covariances(n_clouds, n) if covariances else (None, None, None)
    ok = [r for r in res if r.status == 0]
    out = JointResult(H, table, max((int(r.iterations) for r in ok), default=0),
                      bool(ok) and all(bool(r.converged) for r in ok), results, *cov,
                      relative_misclosure(H, relative_pairs, relative_poses) if rel else None)
    _raise_failed(table, on_error, messages, results)
    return out


def _joint_priors(prior_poses, prior_weights, free: np.ndarray):
    """simpleicp_joint's pose priors checked: (poses, weights, full) as float64 arrays of shapes
    (n_clouds, 4, 4) and (n_clouds, 6), and the mask of the free clouds whose six weights are all
    > 0.  Every weight must be finite and >= 0; the pose of a read prior (a free cloud with a
    non-zero weight) finite and rigid to 1e-6.  Else ValueError."""
    n_clouds = free.shape[0]
    W = np.ascontiguousarray(prior_weights, dtype=np.float64)
    if W.shape != (n_clouds, 6):
        raise ValueError(f"prior_weights must have shape ({n_clouds}, 6), got {W.shape}")
    if not np.isfinite(W).all() or (W < 0).any():
        raise ValueError("prior_weights must be finite and >= 0 (a cloud whose pose is exact belongs in fixed)")
    P = np.ascontiguousarray(prior_poses, dtype=np.float64)
    if P.shape != (n_clouds, 4, 4):
        raise ValueError(f"prior_poses must have shape ({n_clouds}, 4, 4), got {P.shape}")
    read = free & (W != 0).any(axis=1)
    bad = read & ~np.isfinite(P).all(axis=(1, 2))
    if bad.any():
        raise ValueError(f"prior_poses[{int(np.flatnonzero(bad)[0])}] has non-finite entries")
    try:
        _check_rigid(P[read])
    except ValueError as ex:
        raise ValueError(f"prior_poses: {ex}") from None
    return P, W, read & (W > 0).all(axis=1)


def _joint_relative(pairs, poses, weights, used: np.ndarray, free: np.ndarray):
    """simpleicp_joint's relative observations checked: (pairs, poses, weights, link) as an int64
    (n_rel, 2) array and float64 arrays of shapes (n_rel, 4, 4) and (n_rel, 6), and the mask of the
    observations whose six weights are all > 0 and that are read.  At most 65 535 observations, each
    of two different clouds that edges reference; every weight finite and >= 0; the pose of a read
    observation (a non-zero weight, a free cloud) finite and rigid to 1e-6.  Else ValueError."""
    n_clouds = free.shape[0]
    p = np.asarray(pairs)
    if p.ndim != 2 or p.shape[1] != 2 or not np.issubdtype(p.dtype, np.integer):
        raise ValueError(f"relative_pairs must be integers of shape (n_rel, 2), got {p.dtype} of shape {p.shape}")
    p = p.astype(np.int64)
    n = p.shape[0]
    if n > 65535:
        raise ValueError(f"at most 65535 relative observations, got {n}")
    if n and (p.min() < 0 or p.max() >= n_clouds):
        raise ValueError(f"relative_pairs must index the {n_clouds} clouds")
    if np.any(p[:, 0] == p[:, 1]):
        k = int(np.flatnonzero(p[:, 0] == p[:, 1])[0])
        raise ValueError(f"relative_pairs must join two clouds: observation {k}")
    bad = ~(used[p[:, 0]] & used[p[:, 1]])
    if bad.any():
        raise ValueError(f"relative observation {int(np.flatnonzero(bad)[0])} joins a cloud that no edge references")
    W = np.ascontiguousarray(weights, dtype=np.float64)
    if W.shape != (n, 6):
        raise ValueError(f"relative_weights must have shape ({n}, 6), got {W.shape}")
    if not np.isfinite(W).all() or (W < 0).any():
        raise ValueError("relative_weights must be finite and >= 0")
    Z = np.ascontiguousarray(poses, dtype=np.float64)
    if Z.shape != (n, 4, 4):
        raise ValueError(f"relative_poses must have shape ({n}, 4, 4), got {Z.shape}")
    read = (W != 0).any(axis=1) & (free[p[:, 0]] | free[p[:, 1]])
    bad = read & ~np.isfinite(Z).all(axis=(1, 2))
    if bad.any():
        raise ValueError(f"relative_poses[{int(np.flatnonzero(bad)[0])}] has non-finite entries")
    try:
        _check_rigid(Z[read])
    except ValueError as ex:
        raise ValueError(f"relative_poses: {ex}") from None
    return p, Z, W, read & (W > 0).all(axis=1)


def _rotvec(M: np.ndarray) -> np.ndarray:
    """The rotation vectors (n, 3) of rotations M (n, 3, 3), angles in [0, pi]: the axis from the
    skew part below 2 pi / 3, else from the symmetric part, as the device's rotvec."""
    s = 0.5 * np.stack((M[:, 2, 1] - M[:, 1, 2], M[:, 0, 2] - M[:, 2, 0], M[:, 1, 0] - M[:, 0, 1]), axis=1)
    sn = np.linalg.norm(s, axis=1)
    cs = 0.5 * (np.trace(M, axis1=1, axis2=2) - 1.0)
    th = np.arctan2(sn, cs)
    with np.errstate(invalid="ignore", divide="ignore"):
        w = s * np.where(sn > 0.0, th / sn, 1.0)[:, None]
    for i in np.flatnonzero(cs <= -0.5):
        k = int(np.argmax(np.diagonal(M[i])))
        n = 0.5 * (M[i][:, k] + M[i][k, :])
        n[k] = M[i][k, k] - cs[i]
        n *= np.copysign(1.0, n @ s[i]) / np.sqrt(n[k] * (1.0 - cs[i]))
        w[i] = th[i] * n
    return w


def relative_misclosure(H, pairs, Z) -> np.ndarray:
    """(n_rel, 6): each relative observation's (rotvec(R_Z R_ab^T), t_Z - t_ab) at the poses H
    (n_clouds, 4, 4), R_ab = R_a^T R_b and t_ab = R_a^T (o_b - o_a) (DESIGN.md §6.13)."""
    H = np.asarray(H, dtype=np.float64)
    Z = np.asarray(Z, dtype=np.float64).reshape(-1, 4, 4)
    pairs = np.asarray(pairs, dtype=np.int64).reshape(-1, 2)
    Ra, Rb = H[pairs[:, 0], :3, :3], H[pairs[:, 1], :3, :3]
    Rab = np.transpose(Ra, (0, 2, 1)) @ Rb
    tab = np.einsum("nji,nj->ni", Ra, H[pairs[:, 1], :3, 3] - H[pairs[:, 0], :3, 3])
    return np.concatenate((_rotvec(Z[:, :3, :3] @ np.transpose(Rab, (0, 2, 1))), Z[:, :3, 3] - tab), axis=1)


def _check_edges(edges, n_clouds: int) -> np.ndarray:
    """edges as an (n_edges, 2) int64 array of indices into n_clouds clouds, or ValueError."""
    e = np.asarray(edges)
    if e.ndim != 2 or e.shape[1] != 2:
        raise ValueError(f"edges must have shape (n_edges, 2), got {e.shape}")
    if e.size and not np.issubdtype(e.dtype, np.integer):
        raise ValueError(f"edges must hold integer cloud indices, got {e.dtype}")
    e = e.astype(np.int64)
    if e.size and (e.min() < 0 or e.max() >= n_clouds):
        raise ValueError(f"edges must index the {n_clouds} clouds: every entry in [0, {n_clouds})")
    return e


def edge_chunks(edges: np.ndarray, mine: Sequence[int], batch_size: int):
    """The library calls of simpleicp_edges for a rank's share `mine` (edge numbers, in order):
    `batch_size` edges per call, in order.  Each call is (js, cloud_ids, local_edges): the positions
    js in `mine` of its edges, the clouds it passes (ascending indices into the caller's clouds:
    exactly those its edges reference) and its edges remapped to positions in cloud_ids, so that
    cloud_ids[local_edges[k]] == edges[mine[js[k]]]."""
    bs = max(1, int(batch_size))
    out = []
    for lo in range(0, len(mine), bs):
        js = np.arange(lo, min(lo + bs, len(mine)))
        cloud_ids, inv = np.unique(edges[np.asarray(mine, dtype=np.int64)[js]], return_inverse=True)
        out.append((js, cloud_ids, inv.reshape(-1, 2)))
    return out


_BATCH_KEYS = {"correspondences", "neighbors", "min_planarity", "min_change", "max_iterations",
               "distance_weights", "rbp_observed_values", "rbp_observation_weights", "max_overlap_distance",
               "want_normals", "mov_neighbors", "max_angle_between_normals"}
# run() arguments simpleicp_edges (sicp_register_pairs) and Map.register (sicp_register_to_map)
# serve: the batched engine's, without the debug output
_EDGE_KEYS = _MAP_KEYS = _BATCH_KEYS - {"want_normals"}
# the batched engines run one block per pair, which holds at most this many correspondences
_MAX_CORRESPONDENCES = 4096


def _batchable(kw) -> bool:
    """Can the batched engine serve these run() arguments?  (One block per pair: at most
    _MAX_CORRESPONDENCES; nothing that needs per-pair host interaction.)"""
    if set(kw) - _BATCH_KEYS:
        return False
    return int(kw.get("correspondences", 1000)) <= _MAX_CORRESPONDENCES and not kw.get("want_normals", False)


def _check_run_keys(kw, allowed, caller: str, unit: str) -> None:
    """The run() arguments of `caller`, which runs one block per `unit` (edge, scan): a key
    outside `allowed` is a TypeError, more than _MAX_CORRESPONDENCES a ValueError."""
    unknown = set(kw) - allowed
    if unknown:
        raise TypeError(f"{caller}() got unsupported arguments {sorted(unknown)}")
    if int(kw.get("correspondences", 1000)) > _MAX_CORRESPONDENCES:
        raise ValueError(f"{caller} runs one block per {unit}: correspondences must be <= {_MAX_CORRESPONDENCES}")


def _check_mov_kwargs(kw) -> None:
    """mov_neighbors / max_angle_between_normals checked as register() checks them (the movable
    point counts are checked per pair where the clouds are)."""
    from .simpleicp import _check_mov_arguments

    _check_mov_arguments(kw.get("mov_neighbors"), kw.get("max_angle_between_normals"), kw.get("mov_normals"))


def _per_pair_observed(kw, n_pairs: int):
    """rbp_observed_values given per pair: the (n_pairs, 6) rows as float64 (degrees), each
    checked as run() checks the common tuple.  None when the common 6-tuple (or nothing) is given."""
    from .simpleicp import SimpleICPException, _check_arguments

    if "rbp_observed_values" not in kw:
        return None
    try:
        v = np.asarray(kw["rbp_observed_values"], dtype=np.float64)
    except (TypeError, ValueError):
        v = None
    if v is not None and v.ndim == 1:
        return None  # the common tuple: checked where it is used, as before
    if v is None or v.shape != (n_pairs, 6):
        raise SimpleICPException(
            f"rbp_observed_values must have exactly 6 elements, or shape ({n_pairs}, 6) for one row per pair.")
    for row in v:
        _check_arguments(kw.get("distance_weights", 1), row, kw.get("rbp_observation_weights", (0.0,) * 6))
    if not np.isfinite(v).all():
        raise SimpleICPException("Every row of rbp_observed_values must be finite.")
    return v


_BATCH_ENGINES: dict = {}


def _batch_engine(device: int):
    """The batched engine kept for `device` in _BATCH_ENGINES, created when missing or closed;
    called under torch.cuda.device(device)."""
    from . import _capi

    eng = _BATCH_ENGINES.get(int(device))
    if eng is None or not eng.alive:
        eng = _BATCH_ENGINES[int(device)] = _capi.Engine(int(device))
    return eng


def _run_batched(get, mine, local, device, batch_size, kw, messages, rows=None, map_engine=None, results=None,
                 edges=None):
    """The rank's share `mine` through the batched engine, `batch_size` pairs per call, records into
    `local`.  With `map_engine` (an engine holding a map, sicp_set_map) get(i) is scan i alone and
    every chunk is registered against that map (sicp_register_to_map).  With `edges` (n_edges x 2
    cloud indices) get(i) is cloud i, pair i is edge i, and every chunk passes the clouds its edges
    reference (edge_chunks, sicp_register_pairs).  With `results` (a list of
    len(mine)) the full output of every pair that succeeded goes there too, fetched after each call
    (sicp_get_batch_outputs) because the next one reuses the library's buffers."""
    import torch

    from .simpleicp import _check_arguments, _observed_in_radians

    dw = kw.get("distance_weights", 1)
    obs_w = kw.get("rbp_observation_weights", (0.0,) * 6)
    if rows is None:
        obs_v = kw.get("rbp_observed_values", (0.0,) * 6)
        _check_arguments(dw, obs_v, obs_w)
        obs = _observed_in_radians(obs_v)
    else:
        obs = np.zeros(6)  # every pair's x0 and observed values come from its row
    mod = float(kw.get("max_overlap_distance", np.inf))
    k_mov = kw.get("mov_neighbors")
    ang = kw.get("max_angle_between_normals")
    with torch.cuda.device(device):
        # a closed map's engine is replaced too: the call then reports that there is no map
        eng = map_engine if map_engine is not None and map_engine.alive else _batch_engine(device)
        register = eng.register_to_map if map_engine is not None else eng.register_batch
        lsq = eng.lsq_params(obs, obs, [float(w) for w in obs_w], dw)
        params = eng.run_params(kw.get("min_planarity", 0.3), kw.get("min_change", 1.0),
                                kw.get("max_iterations", 100), lsq)
        bs = max(1, int(batch_size))
        chunks = (edge_chunks(edges, mine, bs) if edges is not None else
                  [(range(lo, min(lo + bs, len(mine))), None, None) for lo in range(0, len(mine), bs)])
        for ids, cloud_ids, local_edges in chunks:
            observed = None if rows is None else np.array([_observed_in_radians(rows[mine[j]]) for j in ids])
            args = (kw.get("correspondences", 1000), kw.get("neighbors", 10), params, mod if np.isfinite(mod) else -1.0,
                    observed, 0 if k_mov is None else int(k_mov), -1.0 if ang is None else float(np.deg2rad(ang)))
            if edges is None:
                res = register([get(mine[j]) for j in ids], *args)
            else:
                res = eng.register_pairs([get(int(c)) for c in cloud_ids], local_edges, *args)
            for j, r in zip(ids, res):
                local[j] = _pair_record(r, "pair", mine[j], messages)
            if results is not None:
                for k, (j, r, o) in enumerate(zip(ids, res, eng.batch_outputs(res))):
                    if o is not None:
                        results[j] = _batch_result(r, o, obs if observed is None else observed[k], obs_w)


def _batch_result(r, outputs, obs, rbp_observation_weights):
    """register()'s result object for one pair of a batched call: its PairResult `r` and its
    sicp_get_batch_outputs part `outputs`; `obs` is the pair's prior in radians."""
    from .simpleicp import _make_rbp, _records, _Result

    X_t, residuals, log, _ = outputs
    records, iterations = _records(log), int(r.iterations)
    res = _Result()
    res.H = np.array(r.H).reshape(4, 4)
    res.X_mov_transformed, res.residuals, res.records = X_t, residuals, records
    res.rbp = _make_rbp(obs, rbp_observation_weights, records, iterations, np.array(r.x), np.array(r.sigma))
    res.iterations, res.converged = iterations, bool(r.converged)
    res.idx_selected = res.normals = res.timings = res.loop_ms = res.initial_stats = None
    return res


def _finite_array(a, name: str, shape: tuple) -> np.ndarray:
    """`a` as a float64 array of `shape` with only finite entries, or ValueError."""
    a = np.asarray(a, dtype=np.float64)
    if a.shape != shape:
        raise ValueError(f"{name} must have shape {shape}, got {a.shape}")
    if not np.isfinite(a).all():
        raise ValueError(f"{name} must be finite")
    return a


def _map_clouds(method: str, clouds, H):
    """The `clouds` and `H` of Map.insert / distances / carve checked: at least one cloud, each
    (n, 3), and H None or finite of shape (n_clouds, 4, 4).  Returns (list of clouds, H as
    float64); ValueError otherwise."""
    clouds = list(clouds)
    if not clouds:
        raise ValueError(f"{method} needs at least one cloud")
    for i, X in enumerate(clouds):
        if len(getattr(X, "shape", ())) != 2 or X.shape[1] != 3:
            raise ValueError(f"cloud {i} must have shape (n, 3), got {tuple(getattr(X, 'shape', ()))}")
    return clouds, None if H is None else _finite_array(H, "H", (len(clouds), 4, 4))


def _check_rigid(H: np.ndarray) -> None:
    """ValueError unless every H[i] has the bottom row (0, 0, 0, 1) and an orthonormal rotation
    part (|R^T R - I| <= 1e-6 entrywise), as sicp_overlap_graph requires."""
    if np.any(H[:, 3, :] != np.array([0.0, 0.0, 0.0, 1.0])):
        raise ValueError("H must have the bottom row (0, 0, 0, 1)")
    R = H[:, :3, :3]
    if np.abs(np.einsum("nji,njk->nik", R, R) - np.eye(3)).max(initial=0.0) > 1e-6:
        raise ValueError("the rotation part of H must be orthonormal (to 1e-6)")


@dataclass
class OverlapGraph:
    """overlap_graph's result: one row per pair (a, b), a < b, of clouds that overlap under the
    poses, ascending.  ``pairs`` (m, 2) int64; ``counts`` (m, 2) int64 [count_ab, count_ba], the
    sampled points of a within max_distance of b and the other way round; ``sampled`` (n_clouds,)
    int64 the points each cloud samples, ceil(n_c / stride); ``fraction`` (m, 2) float64 each count
    over the sampled points of its source cloud (a for count_ab, b for count_ba)."""

    pairs: np.ndarray
    counts: np.ndarray
    sampled: np.ndarray
    fraction: np.ndarray


def overlap_graph(clouds: Sequence, H=None, *, max_distance: float, stride: int = 1, device: int = 0) -> OverlapGraph:
    """Which pairs of these clouds overlap under these poses, and by how much (sicp_overlap_graph).

    ``clouds`` is a sequence of (n_i, 3) NumPy arrays or CUDA tensors (empty clouds take part in
    no pair); ``H`` is None (every cloud already in one frame) or (n_clouds, 4, 4) rigid poses,
    world <- cloud, e.g. GNSS/INS or odometry priors.  For every ordered pair (a, b), count_ab is
    the number of points of ``X_a[::stride]`` whose squared distance to the nearest point of b,
    under T_ab = H_a^-1 H_b, is below max_distance^2: the ``n_kept`` of the pair's overlap filter
    (fixed a, movable b, prior T_ab).  A pair is reported when count_ab + count_ba > 0.  The rows
    make the edges of ``simpleicp_joint`` or ``simpleicp_edges``, e.g.
    ``g.pairs[g.fraction.min(axis=1) > 0.2]``.  One library call on one device."""
    r = float(max_distance)
    if not (np.isfinite(r) and r > 0):
        raise ValueError(f"max_distance must be finite and > 0, got {max_distance}")
    if isinstance(stride, (bool, np.bool_)) or int(stride) != stride or not 1 <= int(stride) < (1 << 63):
        raise ValueError(f"stride must be an integer >= 1, got {stride}")
    s = int(stride)
    clouds, H = _map_clouds("overlap_graph", clouds, H)
    if H is not None:
        _check_rigid(H)
    n = np.array([int(X.shape[0]) for X in clouds], dtype=np.int64)
    if int(n.sum()) >= 1 << 32:
        raise ValueError("the points of the clouds must be below 2^32")
    sampled = (n + s - 1) // s
    import torch

    with torch.cuda.device(device):
        eng = _batch_engine(device)
        cap = 8 * len(clouds)
        total, pairs, counts = eng.overlap_graph(clouds, H, max_distance=r, stride=s, cap=cap)
        if total > cap:  # the second call recomputes everything, with room for every row
            total, pairs, counts = eng.overlap_graph(clouds, H, max_distance=r, stride=s, cap=total)
    # a reported pair's clouds are not empty: every divisor is >= 1
    return OverlapGraph(pairs, counts, sampled, counts / sampled[pairs])


class Map:
    """A fixed cloud (a map) held on one GPU, against which many scans are registered.

    ``Map(X_map, device=0)`` uploads the map and builds its search grid once.  Each call of
    ``register(scans, ...)`` then registers every scan against it with the batched engine
    (sicp_register_to_map), ``batch_size`` scans per library call: the map is neither uploaded
    nor gridded again, and with ``max_overlap_distance`` the overlap filter only searches the map
    points near each scan (under its prior), so the work per scan grows with its footprint, not
    with the map.  Scan i's result is that of
    ``register(X_map, scans[i], rbp_observed_values=row_i, max_overlap_distance=d, ...)``.
    ``insert(clouds, H, voxel_size=v)`` grows the map on the device by what the scans saw (one
    new point per voxel the map does not occupy) and ``points()`` reads it back.
    ``distances(clouds, H, max_distance=d)`` tells how well clouds fit the map: every point's
    nearest map point within d, with fitness and inlier RMSE per cloud.
    ``crop(centers, radius=R)`` shrinks the map on the device to the points within R of the given
    positions (a local map around the sensor, so a loop that keeps inserting stays bounded), and
    ``thin(voxel_size=v)`` to one point per voxel (a dense base map); both keep the points' order
    and leave a map that registers as ``Map(points)`` of the same points would.
    ``carve(clouds, H, radius=r, margin=e)`` removes what the scans' rays see through (free
    space), the same way.
    """

    def __init__(self, X_map, device: int = 0):
        import torch

        from . import _capi

        self.device = int(device)
        with torch.cuda.device(self.device):
            self._engine = _capi.Engine(self.device)
            self._engine.set_map(X_map)
        self.n_points = self._engine.n_map

    def register(self, scans: Sequence[np.ndarray], *, batch_size: int = 64, on_error: str = "raise",
                 full_output: bool = False, **run_kwargs):
        """Register every scan against the map; returns the (n_scans, 20) record table of
        simpleicp_batch.  ``run_kwargs`` are SimpleICP.run's arguments the batched engine serves
        (at most 4096 correspondences); ``rbp_observed_values`` is the common 6-tuple or one row
        per scan (degrees), each scan's prior.  A scan that cannot be registered (no overlap with
        the map, too few correspondences) gets a NaN record whose ``iterations`` field is minus
        the library's status code; ``on_error="raise"`` then raises BatchError with the full
        table, ``on_error="nan"`` returns it.  ``full_output=True`` returns ``(table, results)``
        as simpleicp_batch does: ``results[i]`` is register()'s result object for scan i
        (``X_mov_transformed`` in the map's frame, residuals, records, uncertainties), None for
        a scan that failed."""
        _check_run_keys(run_kwargs, _MAP_KEYS, "Map.register", "scan")
        n = len(scans)
        rows = _per_pair_observed(run_kwargs, n)
        _check_mov_kwargs(run_kwargs)
        local = np.zeros((n, RECORD_LEN))
        results = [None] * n if full_output else None
        messages: List[str] = []
        # the survivor offsets of one call are 32-bit: scans per call x map points < 2^32
        per_call = max(1, min(int(batch_size), ((1 << 32) - 1) // max(self.n_points, 1)))
        _run_batched(lambda i: scans[i], list(range(n)), local, self.device, per_call, run_kwargs, messages, rows,
                     map_engine=self._engine, **({"results": results} if full_output else {}))
        _raise_failed(local, on_error, messages, results)
        return (local, results) if full_output else local

    def insert(self, clouds, H=None, *, voxel_size: float) -> np.ndarray:
        """Grow the map on the device: for every voxel of edge ``voxel_size`` the map does not
        occupy, append the first new point that falls into it (sicp_map_insert).

        ``clouds`` is a sequence of (n_i, 3) NumPy arrays or CUDA tensors, taken in order; ``H``
        is None or an (n_clouds, 4, 4) array moving cloud i into the map's frame first, e.g.
        ``table[:, :16].reshape(-1, 4, 4)`` of the scans ``register`` registered.  A voxel is the
        key floor(p / voxel_size) per axis; points with a NaN or inf coordinate are skipped.  The
        map keeps its points and order and gets the added ones at its end, and registers as
        ``Map(points)`` of the same points would.  Returns the number of points each cloud added
        (int64)."""
        v = float(voxel_size)
        if not (np.isfinite(v) and v > 0):
            raise ValueError(f"voxel_size must be finite and > 0, got {voxel_size}")
        clouds, H = _map_clouds("insert", clouds, H)
        import torch

        with torch.cuda.device(self.device):
            added = self._engine.map_insert(clouds, H, voxel_size=v)
        self.n_points = self._engine.n_map
        return added

    def distances(self, clouds, H=None, *, max_distance: float, neighbors: Optional[int] = None
                  ) -> List["CloudDistances"]:
        """How well each cloud fits the map: the nearest map point of every point within
        ``max_distance`` (sicp_map_distances), one CloudDistances per cloud.

        ``clouds`` and ``H`` are as in ``insert``.  The rows of the table ``register`` returns for
        the scans that registered plug in: with ``ok = [i for i in range(len(scans)) if t[i, 16] > 0]``,
        ``m.distances([scans[i] for i in ok], t[ok, :16].reshape(-1, 4, 4), max_distance=0.5)``
        (a scan that failed has a NaN H, which is refused).  A point is within
        when its squared distance to the nearest map point is below max_distance^2 (cKDTree's
        ``distance_upper_bound``); ties go to the lower map index.  ``neighbors`` = k also gives
        the signed distance along the matched map point's normal and its planarity, estimated from
        the k nearest map points as ``estimate_normals(k)`` would with the map as the fixed cloud.
        The search walks about (2 max_distance / h + 1)^3 map cells per point for a map cell size
        h, so the bound is required and finite."""
        r = float(max_distance)
        if not (np.isfinite(r) and r > 0):
            raise ValueError(f"max_distance must be finite and > 0, got {max_distance}")
        k = 0 if neighbors is None else int(neighbors)
        if neighbors is not None and not (2 <= k <= 64 and k <= self.n_points):
            raise ValueError(f"neighbors must be between 2 and 64 and at most the map's {self.n_points} points, "
                             f"got {neighbors}")
        clouds, H = _map_clouds("distances", clouds, H)
        import torch

        with torch.cuda.device(self.device):
            idx, d2, pd, pl, n_within = self._engine.map_distances(clouds, H, max_distance=r, neighbors=k)
        return [CloudDistances.of(idx[i], d2[i], None if pd is None else pd[i], None if pl is None else pl[i],
                                  int(n_within[i])) for i in range(len(clouds))]

    def crop(self, centers, *, radius: float) -> int:
        """Shrink the map on the device to the surroundings of ``centers`` (sicp_map_crop): keep
        the map points within ``radius`` of at least one centre, in their order, e.g.
        ``m.crop(table[ok, :16].reshape(-1, 4, 4)[:, :3, 3], radius=100.0)`` for the positions of
        the scans just registered.  ``centers`` is one (3,) position or an (n, 3) array in the
        map's frame.  Point p is kept iff (dx dx + dy dy) + dz dz < radius^2 for some centre
        (d = p - c, each operation rounded in double).  Returns the number of points removed; a
        crop that would keep no point raises the library's SicpError (code 2,
        SICP_ERR_NO_OVERLAP) and leaves the map as it was."""
        c = np.asarray(centers, dtype=np.float64)
        if c.shape == (3,):
            c = c.reshape(1, 3)
        if c.ndim != 2 or c.shape[1] != 3 or c.shape[0] < 1:
            raise ValueError(f"centers must have shape (3,) or (n, 3) with n >= 1, got {c.shape}")
        if not np.isfinite(c).all():
            raise ValueError("centers must be finite")
        r = float(radius)
        if not (np.isfinite(r) and r > 0):
            raise ValueError(f"radius must be finite and > 0, got {radius}")
        import torch

        with torch.cuda.device(self.device):
            removed = self._engine.map_crop(c, r)
        self.n_points = self._engine.n_map
        return removed

    def thin(self, *, voxel_size: float) -> int:
        """Thin the map on the device to one point per voxel (sicp_map_thin): of the map points
        that share a voxel key floor(p / voxel_size) (``insert``'s key), the first in map order is
        kept.  The kept points keep their order, and later inserts at the same voxel size keep the
        map at one point per voxel.  Meant for a dense base map (``Map(X_tls)``).  Returns the
        number of points removed."""
        v = float(voxel_size)
        if not (np.isfinite(v) and v > 0):
            raise ValueError(f"voxel_size must be finite and > 0, got {voxel_size}")
        import torch

        with torch.cuda.device(self.device):
            removed = self._engine.map_thin(v)
        self.n_points = self._engine.n_map
        return removed

    def carve(self, clouds, H=None, *, origins=None, radius: float, margin: float, min_passes: int = 1,
              return_passes: bool = False):
        """Carve free space out of the map on the device (sicp_map_carve): remove the map points
        that the scans' rays pass, such as a car that has since driven off.

        ``clouds`` and ``H`` are as in ``insert``.  Every finite moved point p of cloud i is a ray
        from the sensor origin o_i, by default H[i]'s translation column (a scan given in its own
        sensor frame was taken there); ``origins`` ((n_clouds, 3), the map's frame) gives them
        explicitly, as clouds already in the map's frame need.  With d = p - o, u = m - o,
        L = sqrt((dx dx + dy dy) + dz dz), s = ((ux dx + uy dy) + uz dz) / L and
        e2 = ((ux ux + uy uy) + uz uz) - s s (each operation rounded in double), the ray passes map
        point m iff L > 0 and finite, 0 < s < L - margin and e2 < radius^2.  A map point that
        ``min_passes`` or more rays of this call pass is removed; the rest keep their order.

        ``margin`` keeps the rays off the surfaces they end on: a ray that meets a surface at an
        angle a passes within ``radius`` of it over about radius / sin(a) before its end, so
        surface points are carved where radius / sin(a) > margin (grazing rays).  ``min_passes`` >
        1 makes a single stray ray harmless.  Returns the number of points removed, and with
        ``return_passes=True`` ``(removed, passes)``: the pass count of every point of the map as
        it was (np.uint32).  A carve that would remove every point raises the library's SicpError
        (code 2, SICP_ERR_NO_OVERLAP) and leaves the map as it was."""
        r, mg = float(radius), float(margin)
        if not (np.isfinite(r) and r > 0):
            raise ValueError(f"radius must be finite and > 0, got {radius}")
        if not (np.isfinite(mg) and mg >= 0):
            raise ValueError(f"margin must be finite and >= 0, got {margin}")
        if isinstance(min_passes, bool) or int(min_passes) != min_passes or not 1 <= int(min_passes) < (1 << 31):
            raise ValueError(f"min_passes must be an integer >= 1, got {min_passes}")
        clouds, H = _map_clouds("carve", clouds, H)
        if origins is not None:
            origins = _finite_array(origins, "origins", (len(clouds), 3))
        elif H is None:
            raise ValueError("carve needs origins, or H whose translations are the sensor origins")
        import torch

        passes = np.zeros(self.n_points, dtype=np.uint32) if return_passes else None
        with torch.cuda.device(self.device):
            removed = self._engine.map_carve(clouds, H, origins=origins, radius=r, margin=mg,
                                             min_passes=int(min_passes), passes=passes)
        self.n_points = self._engine.n_map
        return (removed, passes) if return_passes else removed

    def points(self) -> np.ndarray:
        """The map as it stands, (n_points, 3) float64 in map order (a copy): the points it was
        made of followed by those ``insert`` added, less those ``crop``, ``thin`` and ``carve`` removed.
        ``sb.write_xyz(path, m.points())`` saves it."""
        import torch

        with torch.cuda.device(self.device):
            return self._engine.get_map()

    def close(self) -> None:
        """Release the map and its engine."""
        self._engine.close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


@dataclass
class CloudDistances:
    """One cloud's fit to the map (Map.distances).  Per point: ``index`` of the nearest map point
    within the bound (int64, -1 where there is none), its ``distance`` (sqrt of the squared
    distance: +inf beyond the bound, NaN for a point with a NaN or inf coordinate), and with
    ``neighbors`` the signed ``plane_distance`` along that map point's normal and its
    ``planarity`` (NaN where index is -1; None without ``neighbors``).  Per cloud: ``n_within``,
    ``fitness`` = n_within / n over all n points as Open3D's evaluate_registration counts it (NaN
    for an empty cloud), and ``rmse`` = the root mean square distance of the within points (NaN
    when there are none)."""

    index: np.ndarray
    distance: np.ndarray
    plane_distance: Optional[np.ndarray]
    planarity: Optional[np.ndarray]
    n_within: int
    fitness: float
    rmse: float

    @classmethod
    def of(cls, index, dist2, plane_distance, planarity, n_within: int) -> "CloudDistances":
        index, dist2 = np.asarray(index), np.asarray(dist2, dtype=np.float64)
        n = len(index)
        inside = dist2[index >= 0]
        fitness = n_within / n if n else float("nan")
        rmse = float(np.sqrt(np.mean(inside))) if inside.size else float("nan")
        return cls(index, np.sqrt(dist2), plane_distance, planarity, int(n_within), fitness, rmse)


class BatchError(RuntimeError):
    """Some pairs of a batch could not be registered; `.table` is the complete record table,
    `.results` the per-pair results of a `full_output=True` call (None otherwise)."""

    def __init__(self, table, failed, messages, results=None):
        codes = sorted({int(-table[i, 16]) for i in failed})
        super().__init__(f"{len(failed)} of {len(table)} pairs failed (pairs {failed[:8].tolist()}"
                         f"{' ...' if len(failed) > 8 else ''}, status codes {codes})"
                         + (f"; first local message: {messages[0]}" if messages else ""))
        self.table, self.failed, self.messages, self.results = table, failed, messages, results
