"""simpleicp_batch with one prior per pair and the overlap filter: argument checks, sharding of
the rows, engine choice.  Host only (the registrations are stubs)."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from conftest import REPO

from simpleicp_b200 import batch
from simpleicp_b200.simpleicp import SimpleICPException


def _never(*a, **kw):
    raise AssertionError("no registration may start before the arguments are checked")


def _get(i):
    return np.full((1, 3), float(i)), np.zeros((1, 3))


@pytest.mark.parametrize("obs", [np.zeros((4, 6)), np.zeros((5, 5)), np.zeros((5, 7)), np.zeros((6, 1)),
                                 np.zeros((5, 6, 1)), 0.0, [[0.0] * 6] * 4 + [[0.0] * 5]])
def test_bad_row_shapes_raise_before_any_registration(obs):
    with pytest.raises(SimpleICPException, match="shape"):
        batch.simpleicp_batch(_get, 5, register_fn=_never, rbp_observed_values=obs)
    with pytest.raises(SimpleICPException, match="shape"):  # the GPU engines are never reached either
        batch.simpleicp_batch(_get, 5, rbp_observed_values=obs, max_overlap_distance=1.0)


def test_invalid_rows_raise_before_any_registration():
    rows = np.zeros((5, 6))
    rows[3, 4] = np.nan
    with pytest.raises(SimpleICPException, match="finite"):
        batch.simpleicp_batch(_get, 5, register_fn=_never, rbp_observed_values=rows)
    with pytest.raises(SimpleICPException, match=">= 0"):
        batch.simpleicp_batch(_get, 5, register_fn=_never, rbp_observed_values=np.zeros((5, 6)),
                              rbp_observation_weights=(0, 0, 0, -1, 0, 0))
    with pytest.raises(SimpleICPException, match="distance_weights"):
        batch.simpleicp_batch(_get, 5, rbp_observed_values=np.zeros((5, 6)), distance_weights=-1.0)


def test_common_tuple_still_reaches_every_pair():
    seen = []

    class R:
        H, iterations, records = np.eye(4), 1, [dict(n_kept=10, mean_res=0.0, std_res=0.0)]

    def stub(Xf, Xm, **kw):
        seen.append(kw["rbp_observed_values"])
        return R()

    batch.simpleicp_batch(_get, 3, register_fn=stub, rbp_observed_values=(1, 2, 3, 4, 5, 6))
    assert seen == [(1, 2, 3, 4, 5, 6)] * 3


def test_batchable_accepts_the_overlap_filter():
    assert batch._batchable(dict(max_overlap_distance=0.5, rbp_observed_values=np.zeros((3, 6))))
    assert batch._batchable(dict(max_overlap_distance=np.inf))
    assert not batch._batchable(dict(max_overlap_distance=0.5, correspondences=5000))
    assert not batch._batchable(dict(max_overlap_distance=0.5, want_normals=True))


_GLOO_ROWS = r'''
import sys
sys.path.insert(0, sys.argv[1])
import numpy as np
import torch.distributed as dist
from simpleicp_b200 import batch

class R:
    def __init__(self, i):
        self.H = np.eye(4) * (i + 1); self.iterations = 1
        self.records = [dict(n_kept=i, mean_res=0.0, std_res=0.0)]

dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
n = 7
rows = np.arange(6 * n, dtype=np.float64).reshape(n, 6) - 20.0
got = {}
def stub(Xf, Xm, **kw):
    i = int(Xf[0, 0])
    got[i] = np.asarray(kw["rbp_observed_values"])
    assert kw["max_overlap_distance"] == 0.5
    return R(i)
table = batch.simpleicp_batch(lambda i: (np.full((1, 3), float(i)), np.zeros((1, 3))), n, rank=rank,
                              world_size=world, dist=dist, register_fn=stub, rbp_observed_values=rows,
                              max_overlap_distance=0.5)
assert sorted(got) == batch.shard_pairs(n, world, rank), got
for i, r in got.items():
    assert r.shape == (6,) and np.array_equal(r, rows[i]), (i, r)
assert np.array_equal(table[:, 17], np.arange(n))
dist.destroy_process_group()
print("ok", rank)
'''


def test_rows_follow_their_pairs_under_gloo_world2(tmp_path):
    """world_size 2: each rank hands every pair of its shard that pair's own row."""
    script = tmp_path / "worker.py"
    script.write_text(_GLOO_ROWS)
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
