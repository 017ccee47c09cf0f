"""The narrow-search index copy starts each (probe, block) walk at a directory cell one before the cell of `flo`. tests/narrow_directory.py
restates the host's cell parameters, the directory builder and the probe's start cell with the same binary32 operations; these checks require
the start never to pass the first entry with m/z >= flo (the walk would lose matches silently), on realistic, narrow, wide and near-degenerate
m/z ranges, on flo values exactly on cell edges and one ulp to either side, in the first and last cell, and in blocks whose starts need the
u32 group base (> 65535 entries) or hit the u16 clamp."""
import numpy as np
import pytest

from narrow_directory import F, NARROW_GROUP, build_block, dir_cells, edges, mz_cells, start_cells, walk_start

RANGES = [(57.02146, 4012.37), (100.0, 100.5), (0.0001, 3.0e4), (1.0, 1.0000153), (147.11281, 147.11282), (500.0, 500.0)]


def probes(lo, hi, cells, rng):
    base, inv_w = mz_cells(lo, hi, cells)
    e = edges(base, inv_w, np.arange(1, cells)) if inv_w > 0 else np.zeros(0, F)
    near = np.concatenate([e, np.nextafter(e, F(np.inf)), np.nextafter(e, F(-np.inf))])
    span = max(float(hi) - float(lo), 1e-3)
    rand = rng.uniform(float(lo) - 0.01 * span, float(hi) + 0.01 * span, 200_000).astype(F)
    ends = np.array([lo, hi, np.nextafter(F(lo), F(np.inf)), np.nextafter(F(hi), F(-np.inf)), np.nextafter(F(hi), F(np.inf))], F)
    return base, inv_w, np.concatenate([near, rand, ends]).astype(F)


@pytest.mark.parametrize("cells", [1024, 8192, 32768])
@pytest.mark.parametrize("lo,hi", RANGES)
def test_start_cell_edge_not_above_flo(lo, hi, cells):
    rng = np.random.default_rng(cells)
    base, inv_w, flo = probes(lo, hi, cells, rng)
    c = start_cells(base, inv_w, cells, flo)
    assert c.min() >= 0 and c.max() <= cells - 2
    pos = c > 0
    if pos.any():
        assert np.all(edges(base, inv_w, c[pos]) <= flo[pos])
    if (F(hi) - F(lo)) / cells > 64 * np.spacing(F(hi)):   # cells well above the float spacing: the start is at most two cells early
        c_exact = np.searchsorted(edges(base, inv_w, np.arange(1, cells)), flo, side="right")
        inside = (flo >= F(lo)) & (flo <= F(hi))
        assert np.all(c_exact[inside] - c[inside] <= 2)


def block_mz(kind, n, rng, lo, hi):
    if kind == "uniform":
        return np.sort(rng.uniform(lo, hi, n).astype(F))
    if kind == "clustered":   # most entries on a few hundred masses, as y1 / b2 ions of frequent residues are
        centers = rng.uniform(lo, hi, 300).astype(F)
        return np.sort(np.concatenate([rng.choice(centers, n - n // 4), rng.uniform(lo, hi, n // 4).astype(F)]).astype(F))
    if kind == "one_mass":    # > 65535 entries between two edges of one group: the u16 remainder is clamped
        return np.sort(np.concatenate([np.full(n - 2, F(1234.5678)), np.array([lo, hi], F)]))
    raise ValueError(kind)


@pytest.mark.parametrize("kind,n", [("uniform", 6660), ("uniform", 85_000), ("clustered", 85_000), ("clustered", 200_000), ("one_mass", 70_000),
                                    ("uniform", 0), ("uniform", 1)])
def test_directory_start_not_after_first_match(kind, n):
    rng = np.random.default_rng(n + len(kind))
    lo, hi = F(57.02146), F(4012.37)
    mz = block_mz(kind, n, rng, lo, hi) if n else np.zeros(0, F)
    cells = 32768 if n > 20_000 else 8192
    base, inv_w = mz_cells(lo, hi, cells)
    dir_, grp = build_block(mz, base, inv_w, cells)
    if n > 65535 and kind != "one_mass":
        assert grp.max() > 65535   # the group base carries what 16 bits cannot
    if kind == "one_mass":
        assert dir_.max() == 65535
    flo = np.concatenate([probes(lo, hi, cells, rng)[2], mz, np.nextafter(mz, F(np.inf)), np.nextafter(mz, F(-np.inf))]).astype(F)
    start = walk_start(dir_, grp, start_cells(base, inv_w, cells, flo))
    first = np.searchsorted(mz, flo, side="left")
    assert np.all(start <= first)
    if kind == "uniform" and n:   # and not far before it: at most two cells early, plus the one-cell margin
        assert np.max(first - start) <= 6 * n / cells + 8


def test_dir_cells():
    assert dir_cells(48_900_000, 7330) == 16384       # cfg2: 256-peptide blocks
    assert dir_cells(678_000_000, 8008) == 32768      # cfg3: 2048-peptide blocks, capped
    assert dir_cells(678_000_000, 63_979) == 8192     # cfg3 in blocks of 256 peptides: the 1 GB cap
    assert dir_cells(1000, 50) == 1024 and dir_cells(0, 0) == 1024 and dir_cells(6660, 1) == 16384
    assert 32768 % NARROW_GROUP == 0 and 1024 % NARROW_GROUP == 0
