"""simpleicp_batch(..., full_output=True) on the host paths (stub registrations, a gloo world of
2) and the argument check of sicp_get_batch_outputs that needs no device."""
import os
import re
import socket
import subprocess
import sys

import numpy as np
import pytest

from conftest import REPO

from simpleicp_b200 import _capi, batch


class _Stub:
    """What register_fn returns: enough of register()'s result for the record table."""

    def __init__(self, i):
        self.i = i
        self.H, self.iterations = np.eye(4) * (i + 1), 2
        self.records = [dict(n_kept=0, mean_res=0.0, std_res=0.0), dict(n_kept=10 + i, mean_res=0.5 * i, std_res=0.25)]


def _get(i):
    return np.full((1, 3), float(i)), np.zeros((1, 3))


def _stub(Xf, Xm, **kw):
    i = int(Xf[0, 0])
    if i in (2, 5):
        raise RuntimeError("Point clouds do not overlap within max_overlap_distance")
    return _Stub(i)


def test_full_output_returns_the_objects_of_register_fn_in_pair_order():
    table = batch.simpleicp_batch(_get, 7, register_fn=_stub, on_error="nan")
    t2, results = batch.simpleicp_batch(_get, 7, register_fn=_stub, on_error="nan", full_output=True)
    assert np.array_equal(table, t2, equal_nan=True)
    assert len(results) == 7
    for i, r in enumerate(results):
        if i in (2, 5):
            assert r is None
        else:
            assert isinstance(r, _Stub) and r.i == i
    with pytest.raises(batch.BatchError) as ex:
        batch.simpleicp_batch(_get, 7, register_fn=_stub, full_output=True)
    assert ex.value.failed.tolist() == [2, 5]
    assert [r is None for r in ex.value.results] == [i in (2, 5) for i in range(7)]
    with pytest.raises(batch.BatchError) as ex:
        batch.simpleicp_batch(_get, 7, register_fn=_stub)
    assert ex.value.results is None


_GLOO_FULL = r'''
import sys
sys.path.insert(0, sys.argv[1])
import numpy as np
import torch.distributed as dist
from simpleicp_b200 import batch

class R:
    def __init__(self, i):
        self.i = i
        self.H = np.eye(4) * (i + 1); self.iterations = 1
        self.records = [dict(n_kept=i, mean_res=0.1 * i, std_res=0.0)]

def stub(Xf, Xm, **kw):
    i = int(Xf[0, 0])
    if i == 4:
        raise RuntimeError("Too few correspondences!")
    return R(i)

dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
n = 7
get = lambda i: (np.full((1, 3), float(i)), np.zeros((1, 3)))
plain = batch.simpleicp_batch(get, n, rank=rank, world_size=world, dist=dist, register_fn=stub, on_error="nan")
table, results = batch.simpleicp_batch(get, n, rank=rank, world_size=world, dist=dist, register_fn=stub,
                                       on_error="nan", full_output=True)
assert np.array_equal(plain, table, equal_nan=True)
assert np.array_equal(table[[0, 1, 2, 3, 5, 6], 17], [0, 1, 2, 3, 5, 6]) and table[4, 16] == -3
assert len(results) == n
mine = batch.shard_pairs(n, world, rank)
for i, r in enumerate(results):
    if i in mine and i != 4:
        assert r is not None and r.i == i, (rank, i, r)
    else:
        assert r is None, (rank, i, r)
dist.destroy_process_group()
print("ok", rank)
'''


def test_full_output_under_gloo_world2(tmp_path):
    """world_size 2: the table is the same with and without full_output on every rank, and each
    rank holds result objects for its own share only."""
    script = tmp_path / "worker.py"
    script.write_text(_GLOO_FULL)
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port), str(script), str(REPO)]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count("ok") == 2


def test_getter_rejects_a_null_context():
    lib = _capi.load_library()
    assert lib.sicp_get_batch_outputs(None, 1, None, None, None, None) == _capi.SICP_ERR_BAD_ARG
    assert b"NULL" in lib.sicp_last_error(None)


def test_abi_declares_the_batch_output_entry_point():
    """sicp_get_batch_outputs is an added entry point that changes no struct: the ABI version, the
    map entry points and the sicp_timings layout stay as they were, and the library exports it."""
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION
    assert hasattr(_capi.load_library(), "sicp_get_batch_outputs")
    for name in ("sicp_set_map", "sicp_register_to_map", "sicp_get_batch_outputs"):
        assert re.search(rf"int32_t {name}\(", header) and name in _capi.SYMBOLS
    names = [n for n, _ in _capi.Timings._fields_]
    assert names[-1] == "overlap_candidates" and names[-2] == "mov_normals_ms"
    assert re.search(r"int64_t overlap_candidates;[^}]*\} sicp_timings;", header, re.S)
