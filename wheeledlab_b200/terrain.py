"""Height-field terrain for the Elevation task.

The reference loads ``Terrains/huge_compact.usd`` (a 726 900-triangle mesh: a slab with top at z = 0.2 over
+-20.5 m carrying ramps/boxes up to z = 2.0, slopes mostly 15-25 deg; SURVEY Appendix A.4/C) and collides /
ray-casts against the triangles.  The fused path works on a regular raster of the TOP surface (what a vertical
ray from z+20 hits): ``procedural_heightfield`` synthesises a terrain with the same envelope (BASELINE config 3
says "procedural terrain"); a raster of the real mesh can be passed instead (same array contract).

Array contract: float32 [ny, pitch] with pitch = nx rounded up to a multiple of 4 (TMA needs 16-byte row strides);
sample (ix, iy) is the height at (x0 + ix*cell, y0 + iy*cell).
"""
from __future__ import annotations

import math

import numpy as np


def reference_heightfield():
    """Raster of the reference's own terrain mesh (Terrains/huge_compact.usd, top surface, 0.1 m, 411x411), produced by
    tools/rasterize_terrain.py from the binary USD (pure-Python USDC reader in tools/usdc_read.py) and shipped as a 58 KB
    data file.  Returns (heights [ny, nx] float32, x0, y0, cell).  Spot heights match SURVEY 8c:
    z(0,0)=0.2, z(5.3,-7.7)=0.38109, z(-12.2,3.3)=0.47669; the four 0.5 m corners are outside the mesh (0 = ground plane)."""
    from pathlib import Path
    d = np.load(Path(__file__).resolve().parent / "data" / "terrain_huge_compact_0p1m.npz")
    return d["heights"].astype(np.float32), float(d["x0"]), float(d["y0"]), float(d["cell"])


def pad_pitch(h: np.ndarray) -> np.ndarray:
    ny, nx = h.shape
    pitch = (nx + 3) & ~3
    out = np.zeros((ny, pitch), dtype=np.float32)
    out[:, :nx] = h
    if pitch > nx:
        out[:, nx:] = h[:, -1:]
    return out


def procedural_heightfield(seed: int = 0, half_extent: float = 20.5, cell: float = 0.1, base: float = 0.2, z_max: float = 2.0,
                           n_ramps: int = 28, n_boxes: int = 24):
    """Returns (heights [ny, nx] float32, x0, y0, cell)."""
    n = int(round(2 * half_extent / cell)) + 1
    xs = -half_extent + cell * np.arange(n, dtype=np.float64)
    X, Y = np.meshgrid(xs, xs, indexing="xy")            # X[iy, ix]
    h = np.full((n, n), base, dtype=np.float64)
    rng = np.random.default_rng(seed + 0x7E44A1)
    for _ in range(n_ramps):                              # wedge: rises along `dir` with a 15-25 deg slope, flat top, falls back
        cx, cy = rng.uniform(-17, 17, 2)
        ang = rng.uniform(0, 2 * math.pi)
        slope = math.tan(math.radians(rng.uniform(15, 25)))
        top = rng.uniform(0.3, z_max - base)
        width = rng.uniform(1.0, 3.0)
        plateau = rng.uniform(0.5, 2.5)
        u = (X - cx) * math.cos(ang) + (Y - cy) * math.sin(ang)          # along
        v = -(X - cx) * math.sin(ang) + (Y - cy) * math.cos(ang)         # across
        run = top / slope
        prof = np.clip(np.minimum(u + run + plateau / 2, -(u - run - plateau / 2)) * slope, 0.0, top)
        side = np.clip((width / 2 - np.abs(v)) * 2.0, 0.0, 1.0)          # 0.5 m soft shoulders
        h = np.maximum(h, base + prof * side)
    for _ in range(n_boxes):                              # low platforms with 45 deg chamfers
        cx, cy = rng.uniform(-18, 18, 2)
        sx, sy = rng.uniform(0.6, 2.5, 2)
        top = rng.uniform(0.05, 0.4)
        d = np.minimum(sx / 2 - np.abs(X - cx), sy / 2 - np.abs(Y - cy))
        h = np.maximum(h, base + np.clip(d + top, 0.0, top))
    h = np.clip(h, 0.0, z_max)
    return h.astype(np.float32), -half_extent, -half_extent, cell


def traversability_map(seed: int = 0, map_size=(500, 500), env_size=(100, 100), sub_group_size=(50, 50), num_walkers: int = 1):
    """Black/white traversability map of the Visual task: restates generated_colored_plane / generate_env_map /
    generate_path (visual/utils/__init__.py:8-139; parameters visual/mushr_visual_env_cfg.py:66-90): per 100x100 block,
    one start point per 50x50 sub-group, `num_walkers` random monotone lattice paths to random free cells, then a
    one-step dilation with the asymmetric structure [[0,1,0],[0,1,1],[0,0,0]].  Returns bool [rows, cols]."""
    rng = np.random.default_rng(seed + 0x51A1)
    rows, cols = map_size
    er, ec = env_size
    gr, gc = sub_group_size
    if rows % er or cols % ec:
        raise ValueError("Map size must be a multiple of the sub environment size.")
    m = np.zeros((rows, cols), dtype=bool)
    for bi in range(rows // er):
        for bj in range(cols // ec):
            blk = np.zeros((er, ec), dtype=bool)
            starts = [(int(rng.integers(0, gr)) + i * gr, int(rng.integers(0, gc)) + j * gc)
                      for i in range(er // gr) for j in range(ec // gc)]
            for sr, sc in starts:
                for _ in range(num_walkers):
                    tr, tc = int(rng.integers(0, er)), int(rng.integers(0, ec))
                    while blk[tr, tc]:
                        tr, tc = int(rng.integers(0, er)), int(rng.integers(0, ec))
                    moves = [(-1 if tr < sr else 1, 0)] * abs(tr - sr) + [(0, -1 if tc < sc else 1)] * abs(tc - sc)
                    r, c = sr, sc
                    blk[r, c] = True
                    for k in rng.permutation(len(moves)):
                        r, c = r + moves[k][0], c + moves[k][1]
                        blk[r, c] = True
            m[bi * er:(bi + 1) * er, bj * ec:(bj + 1) * ec] = blk
    from scipy.ndimage import binary_dilation
    return binary_dilation(m, structure=np.array([[0, 1, 0], [0, 1, 1], [0, 0, 0]], dtype=bool), iterations=1)


def pack_traversability(m: np.ndarray) -> np.ndarray:
    """Device blob for the visual task (include/wheeledlab_b200.h): int32 trav_cells[n] | pad to 16 B | uint8 map."""
    m = np.ascontiguousarray(m, dtype=bool)
    ys, xs = m.nonzero()                                   # generate_random_poses: candidates = map.nonzero()
    cells = (ys.astype(np.int64) * m.shape[1] + xs).astype(np.int32)
    off = (cells.size * 4 + 15) & ~15
    blob = np.zeros(off + m.size, dtype=np.uint8)
    blob[: cells.size * 4] = cells.view(np.uint8)
    blob[off:] = m.reshape(-1).astype(np.uint8)
    return blob, int(cells.size)
