"""The phase stamps of the one-pair match (option match_stamps, sicp_get_match_phase_times,
DESIGN §3.2): a diagnostic that must not change what the match computes."""
from __future__ import annotations

import numpy as np
import pytest

from simpleicp_b200 import _capi
from test_gpu_nn_exact import _same


@pytest.mark.gpu
def test_stamps_change_nothing_and_are_ordered(gpu):
    import simpleicp_b200 as sb
    from conftest import load_pair

    Xf, Xm = load_pair("dragon")
    out, counts, stamps = [], [], None
    with _capi.Engine() as e:
        for on in (0, 1):
            e.set_option("match_stamps", on)
            r = sb.register(Xf, Xm, engine=e, want_normals=False, min_change=0.0, max_iterations=40)
            out.append((np.array(r.H), r.records, np.array(r.residuals), np.array(r.X_mov_transformed)))
            counts.append(e.match_counts())
            if on:
                stamps = np.array(e.match_phase_times())
        e.set_option("match_stamps", 0)
    _same(out[1], out[0], "dragon with match_stamps")
    assert counts[1] == counts[0] and counts[0] > 0
    for off in (0, 8):
        t = stamps[off:off + 7]
        # entry, wait released and exit are written on every path; the others where the stamping
        # thread's query was answered from its certificate (-1: not written).  Microseconds from
        # the first block's entry, so the last block's may even be negative.
        seen = t[t != -1.0]
        assert t[0] != -1.0 and t[1] != -1.0 and t[6] != -1.0, t
        assert np.all(np.diff(seen) >= 0), t
    assert stamps[0] == 0.0
