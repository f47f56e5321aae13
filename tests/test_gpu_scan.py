"""The library's int32 prefix sums against numpy: the ordered compaction (o2345_compact) and the marching-cubes triangle
offsets (o2345_mc_tri_offsets), on seeded random inputs at sizes around the 1024-element block and past 1024 blocks,
where the block sums themselves take more than one tile."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZES = [1, 1023, 1024, 1025, 1024 ** 2 + 1, 3 * 1024 ** 2 + 17]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.mark.parametrize("n", SIZES)
def test_compact_matches_numpy(dev, n):
    from o2345 import ops
    rng = np.random.default_rng(n)
    flags = (rng.random(n) < rng.uniform(0.05, 0.95)).astype(np.uint8)
    rows, index, count = ops.compact(torch.from_numpy(flags).to(dev))
    kept = np.flatnonzero(flags)
    assert int(count.item()) == kept.size
    np.testing.assert_array_equal(rows.cpu().numpy()[:kept.size], kept)
    want = np.where(flags == 1, np.cumsum(flags, dtype=np.int64) - 1, -1)
    np.testing.assert_array_equal(index.cpu().numpy(), want)


@pytest.mark.parametrize("n", SIZES)
def test_mc_tri_offsets_matches_numpy(dev, n):
    from o2345 import _lib as L, mc_tables, ops
    rng = np.random.default_rng(1000 + n)
    _, _, ntri = mc_tables.tables()
    ntri = np.ascontiguousarray(ntri, dtype=np.uint8)
    cases = rng.integers(0, 256, size=n + 5, dtype=np.uint8)
    cells = rng.integers(0, n + 5, size=n, dtype=np.int32)
    count = int(rng.integers(0, n))                      # count < max_cells: the tail counts zero triangles
    t = lambda a: torch.from_numpy(a).to(dev)
    cases_d, cells_d, ntri_d = t(cases), t(cells), t(ntri)
    count_d = torch.tensor([count], dtype=torch.int32, device=dev)
    offs = torch.empty(n, dtype=torch.int32, device=dev)
    total = torch.empty(1, dtype=torch.int32, device=dev)
    scratch = torch.empty(L.load().o2345_scan_scratch_ints(n), dtype=torch.int32, device=dev)
    L.call("o2345_mc_tri_offsets", ops._p(cases_d, torch.uint8), ops._p(cells_d, torch.int32), ops._p(count_d, torch.int32),
           n, ops._p(ntri_d, torch.uint8), ops._p(offs, torch.int32), ops._p(total, torch.int32),
           ops._p(scratch, torch.int32), ops._stream())
    counts = np.where(np.arange(n) < count, ntri[cases[cells]], 0).astype(np.int64)
    np.testing.assert_array_equal(offs.cpu().numpy(), np.cumsum(counts) - counts)
    assert int(total.item()) == int(counts.sum())
