"""simpleicp_edges without a GPU: its argument checks (all raised before any device work), the
chunking of edges into library calls with their clouds remapped (edge_chunks), and rank sharding."""
import numpy as np
import pytest

import simpleicp_b200 as sb
from simpleicp_b200 import batch as B
from simpleicp_b200.simpleicp import SimpleICPException


def _clouds(n=5):
    return [np.full((10 + j, 3), float(j)) for j in range(n)]


@pytest.mark.parametrize("edges", [np.zeros((3,), dtype=int), np.zeros((3, 3), dtype=int), np.zeros((2, 2, 2), dtype=int)])
def test_edge_shape(edges):
    with pytest.raises(ValueError, match="shape"):
        sb.simpleicp_edges(_clouds(), edges)


@pytest.mark.parametrize("edges", [np.array([[0.0, 1.0]]), np.array([[True, False]])])
def test_edge_dtype(edges):
    with pytest.raises(ValueError, match="integer"):
        sb.simpleicp_edges(_clouds(), edges)


@pytest.mark.parametrize("edges", [[[0, 5]], [[-1, 0]], [[0, 1], [7, 2]]])
def test_edge_range(edges):
    with pytest.raises(ValueError, match="index the 5 clouds"):
        sb.simpleicp_edges(_clouds(), edges)


def test_per_edge_priors_need_one_row_per_edge():
    edges = [[0, 1], [1, 2], [2, 3]]
    with pytest.raises(SimpleICPException, match=r"shape \(3, 6\)"):
        sb.simpleicp_edges(_clouds(), edges, rbp_observed_values=np.zeros((2, 6)))
    with pytest.raises(SimpleICPException, match="finite"):
        rows = np.zeros((3, 6))
        rows[1, 4] = np.nan
        sb.simpleicp_edges(_clouds(), edges, rbp_observed_values=rows)


def test_unknown_keys_and_correspondences():
    with pytest.raises(TypeError, match="want_normals"):
        sb.simpleicp_edges(_clouds(), [[0, 1]], want_normals=True)
    with pytest.raises(TypeError, match="mov_normals"):
        sb.simpleicp_edges(_clouds(), [[0, 1]], mov_normals=None)
    with pytest.raises(ValueError, match="4096"):
        sb.simpleicp_edges(_clouds(), [[0, 1]], correspondences=4097)


def _check_chunks(edges, mine, bs):
    chunks = B.edge_chunks(edges, mine, bs)
    order = np.concatenate([js for js, _, _ in chunks]) if chunks else np.zeros(0, dtype=int)
    assert np.array_equal(order, np.arange(len(mine)))  # every edge once, in order
    for js, cloud_ids, local in chunks:
        assert len(js) <= bs
        assert np.all(np.diff(cloud_ids) > 0)
        want = edges[np.asarray(mine)[js]]
        assert np.array_equal(cloud_ids[local], want)  # each remapped edge names the same clouds
        assert set(cloud_ids.tolist()) == set(want.ravel().tolist())  # exactly the clouds it references
        assert local.min() >= 0 and local.max() < len(cloud_ids)


@pytest.mark.parametrize("bs", [1, 3, 64])
def test_chunks_of_a_chain(bs):
    n = 20
    edges = np.array([(i, i + 1) for i in range(n - 1)] + [(i, i + 2) for i in range(n - 2)] + [(4, 4), (9, 0)])
    _check_chunks(edges, list(range(len(edges))), bs)
    for ws in (2, 3):
        for rank in range(ws):
            _check_chunks(edges, B.shard_pairs(len(edges), ws, rank), bs)


def test_chunks_pass_the_same_arrays():
    clouds = _clouds(6)
    edges = np.array([[5, 0], [0, 5], [2, 2], [3, 1]])
    for js, cloud_ids, local in B.edge_chunks(edges, [0, 1, 2, 3], 3):
        passed = [clouds[c] for c in cloud_ids]
        for j, (f, m) in zip(js, local):
            assert passed[f] is clouds[edges[j, 0]] and passed[m] is clouds[edges[j, 1]]


def test_rank_sharding(monkeypatch):
    """Edge i belongs to rank i % world_size: each rank's library calls carry only its edges, in
    order, and their priors; the ranks' shares partition the edges."""
    n = 11
    clouds = _clouds(n + 1)
    edges = np.array([(i, i + 1) for i in range(n)])
    rows = np.arange(6 * n, dtype=float).reshape(n, 6) / 100.0
    seen = {}

    def fake(get, mine, local, device, batch_size, kw, messages, rows=None, map_engine=None, results=None,
             edges=None):
        for js, cloud_ids, loc in B.edge_chunks(edges, mine, batch_size):
            for j, (f, m) in zip(js, loc):
                assert get(int(cloud_ids[f])) is clouds[edges[mine[j], 0]]
                assert get(int(cloud_ids[m])) is clouds[edges[mine[j], 1]]
                local[j] = B.pack_record(np.eye(4), 1, 1, float(rows[mine[j], 0]), 0.0)
        seen[len(seen)] = list(mine)

    def gather(local, n_pairs, world_size, rank, dist, device):  # the all-gather, one rank's part
        out = np.full((n_pairs, B.RECORD_LEN), np.nan)
        out[B.shard_pairs(n_pairs, world_size, rank)] = local
        return out

    monkeypatch.setattr(B, "_run_batched", fake)
    monkeypatch.setattr(B, "gather_records", gather)
    shares = []
    for rank in range(3):
        t = sb.simpleicp_edges(clouds, edges, rank=rank, world_size=3, batch_size=2, rbp_observed_values=rows)
        assert seen[rank] == list(range(rank, n, 3))
        assert np.array_equal(t[seen[rank], 18], rows[seen[rank], 0])  # this rank's rows, its own priors
        shares += seen[rank]
    assert sorted(shares) == list(range(n))
