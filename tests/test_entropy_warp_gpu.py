"""The warp-wide entropy decoder (every lane of a decoder warp runs the syntax decoder; map cells, context copies and
coefficient emission are split over the lanes) against the host front-end, which runs the same syntax source serially:
a 4 x 4 sub-grid of the benchmark's tiles (1024 x 1024, CTB 32, WPP: 512 sub-streams in flight at once) must decode to
the same planes, byte for byte, before the in-loop filters (coefficients, modes, QpY of the command stream) and after
them (deblocking edges and QpY maps, SAO parameters)."""
import numpy as np
import pytest

import libheif_b200 as lb

pytestmark = pytest.mark.gpu

SIDE = 4


@pytest.fixture(scope="module")
def bench_tiles():
    import bench
    return bench.make_tiles(range(SIDE * SIDE))


def _decode(tiles, device, stage):
    d = lb.Decoder(host_threads=8)
    try:
        d.set_front_end(device)
        d.set_debug_stage(stage)
        d.decode_grid(tiles, cols=SIDE, rows=SIDE)
        return [p.copy() for p in d.planes_host()]
    finally:
        d.close()


@pytest.mark.parametrize("stage", [1, 0], ids=["before_filters", "final"])
def test_bench_subgrid_device_front_end_equals_host(cuda, bench_tiles, stage):
    got = _decode(bench_tiles, True, stage)
    want = _decode(bench_tiles, False, stage)
    assert len(got) == len(want) == 3
    for c in range(3):
        assert got[c].shape == want[c].shape
        assert np.array_equal(got[c], want[c]), f"plane {c}: first diffs {np.argwhere(got[c] != want[c])[:4].tolist()}"
