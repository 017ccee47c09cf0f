"""CPU restatement, in binary32, of the m/z directory of the narrow-search index copy (sage_b200.cu: db_narrow_index, set_mz_cells;
kernels.cuh: k_narrow_dir, narrow_start_cell). The directory only gives a walk its first entry; the walk decides on the exact m/z values, so
the one property that matters is that the start is never after the first entry with m/z >= flo."""
import numpy as np

F = np.float32
NARROW_GROUP = 64
CELLS_PER_ENTRY = 2


def dir_cells(n_frag, n_block):
    per_block = n_frag // n_block if n_block else 0
    cells = 1024
    while cells < 32768 and cells < per_block * CELLS_PER_ENTRY:
        cells <<= 1
    while cells > 1024 and 2 * n_block * cells > 1 << 30:   # at most 1 GB of directory
        cells >>= 1
    return cells


def mz_cells(lo, hi, cells):
    """(base, inv_w) as the host computes them from the index's m/z range."""
    lo, hi = F(lo), F(hi)
    width = F(hi - lo) / F(cells)
    base = lo if (np.isfinite(lo) and lo > 0) else F(0)
    inv_w = F(F(1) / width) if (np.isfinite(width) and width > 0 and lo > 0) else F(0)
    return base, inv_w


def edges(base, inv_w, c):
    """edge(c) = base + c * (1 / inv_w), every operation rounded to binary32 (c > 0)."""
    return (F(base) + np.asarray(c).astype(F) * (F(1) / F(inv_w))).astype(F)


def start_cells(base, inv_w, cells, flo):
    tt = ((np.asarray(flo, F) - F(base)) * F(inv_w)).astype(F)
    with np.errstate(invalid="ignore"):
        return np.where(tt > F(1), np.minimum(tt, F(cells - 1)).astype(np.int64) - 1, 0)


def build_block(mz, base, inv_w, cells):
    """k_narrow_dir for one block (ascending m/z): (dir u16 [cells], grp u32 [cells / NARROW_GROUP])."""
    c = np.arange(cells)
    below = np.zeros(cells, np.int64)
    if inv_w > 0:
        below[1:] = np.searchsorted(mz, edges(base, inv_w, c[1:]), side="left")
    gb = below[(c // NARROW_GROUP) * NARROW_GROUP]
    return np.minimum(below - gb, 65535).astype(np.uint16), below[::NARROW_GROUP].astype(np.uint32)


def walk_start(dir_, grp, c):
    return grp[c // NARROW_GROUP].astype(np.int64) + dir_[c].astype(np.int64)
