#!/usr/bin/env python
"""Rasterise the TOP surface of the reference's elevation terrain (Terrains/huge_compact.usd: 363 388 vertices,
726 900 triangles, +-20.5 m, z in [0, 2]) onto the regular height-field the elevation path consumes: for every raster
sample, z = max over the triangles covering (x, y) of the barycentric height -- what the reference's vertical ray from
z + 20 m hits (SURVEY.md Appendix C).  Needs the reference's assets:

    python tools/rasterize_terrain.py <the reference's source/ directory>

The result is committed as a data file (wheeledlab_b200/data/terrain_huge_compact_0p1m.npz, 58 KB) because the reference
is not part of this repository.
"""
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
from usdc_read import Crate  # noqa: E402

C_SRC = r"""
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
int main(int argc, char** argv) {
    int nv = atoi(argv[3]), nt = atoi(argv[4]), n = atoi(argv[5]);
    double x0 = atof(argv[6]), cell = atof(argv[7]);
    float* P = malloc(sizeof(float) * 3 * nv); int* I = malloc(sizeof(int) * 3 * nt);
    FILE* f = fopen(argv[1], "rb"); if (fread(P, 4, 3 * (size_t)nv, f) != 3 * (size_t)nv) return 1; fclose(f);
    f = fopen(argv[2], "rb"); if (fread(I, 4, 3 * (size_t)nt, f) != 3 * (size_t)nt) return 1; fclose(f);
    float* H = malloc(sizeof(float) * (size_t)n * n);
    for (size_t k = 0; k < (size_t)n * n; ++k) H[k] = -1.0f;               /* -1 = not covered */
    for (int t = 0; t < nt; ++t) {
        const float *a = P + 3 * I[3 * t], *b = P + 3 * I[3 * t + 1], *c = P + 3 * I[3 * t + 2];
        double det = (double)(b[1] - c[1]) * (a[0] - c[0]) + (double)(c[0] - b[0]) * (a[1] - c[1]);
        if (fabs(det) < 1e-12) continue;                                   /* vertical wall / degenerate in xy */
        double xmin = fmin(a[0], fmin(b[0], c[0])), xmax = fmax(a[0], fmax(b[0], c[0]));
        double ymin = fmin(a[1], fmin(b[1], c[1])), ymax = fmax(a[1], fmax(b[1], c[1]));
        int i0 = (int)ceil((xmin - x0) / cell - 1e-9), i1 = (int)floor((xmax - x0) / cell + 1e-9);
        int j0 = (int)ceil((ymin - x0) / cell - 1e-9), j1 = (int)floor((ymax - x0) / cell + 1e-9);
        if (i0 < 0) i0 = 0; if (j0 < 0) j0 = 0; if (i1 > n - 1) i1 = n - 1; if (j1 > n - 1) j1 = n - 1;
        for (int j = j0; j <= j1; ++j) for (int i = i0; i <= i1; ++i) {
            double x = x0 + i * cell, y = x0 + j * cell;
            double l1 = ((double)(b[1] - c[1]) * (x - c[0]) + (double)(c[0] - b[0]) * (y - c[1])) / det;
            double l2 = ((double)(c[1] - a[1]) * (x - c[0]) + (double)(a[0] - c[0]) * (y - c[1])) / det;
            double l3 = 1.0 - l1 - l2;
            if (l1 < -1e-7 || l2 < -1e-7 || l3 < -1e-7) continue;
            float z = (float)(l1 * a[2] + l2 * b[2] + l3 * c[2]);
            if (z > H[(size_t)j * n + i]) H[(size_t)j * n + i] = z;
        }
    }
    f = fopen(argv[8], "wb"); fwrite(H, 4, (size_t)n * n, f); fclose(f);
    return 0;
}
"""


def main(usd, cell=0.1, half=20.5,
         out=HERE.parent / "wheeledlab_b200" / "data" / "terrain_huge_compact_0p1m.npz"):
    crate = Crate(usd)
    pts_field = [f for f in crate.array_fields("default") if f[0] == 24]          # vec3f arrays: extent, normals, points
    int_field = [f for f in crate.array_fields("default") if f[0] == 3]           # int arrays: counts, indices
    cands = [crate.read_vec3f_array(off) for _, _, off in pts_field]
    pts = [a for a in cands if a.shape[0] == 363388][0]
    ints = [crate.read_int_array(off, comp) for _, comp, off in int_field]
    counts = [a for a in ints if a.size == 726900][0]
    idx = [a for a in ints if a.size == 2180700][0]
    assert (counts == 3).all() and idx.min() == 0 and idx.max() == pts.shape[0] - 1
    print("points", pts.shape, "extent", pts.min(0), pts.max(0), "tris", idx.size // 3)
    n = int(round(2 * half / cell)) + 1
    with tempfile.TemporaryDirectory() as td:
        td = Path(td)
        pts.astype("<f4").tofile(td / "p.bin"); idx.astype("<i4").tofile(td / "i.bin")
        (td / "r.c").write_text(C_SRC)
        subprocess.run(["/usr/bin/gcc", "-O2", "-o", str(td / "r"), str(td / "r.c"), "-lm"], check=True)
        subprocess.run([str(td / "r"), str(td / "p.bin"), str(td / "i.bin"), str(pts.shape[0]), str(idx.size // 3), str(n),
                        str(-half), str(cell), str(td / "h.bin")], check=True)
        H = np.fromfile(td / "h.bin", dtype="<f4").reshape(n, n)                  # H[iy, ix]
    print("uncovered samples:", int((H < 0).sum()), " z range", H[H >= 0].min(), H.max())
    H = np.where(H < 0, np.float32(0.0), H)
    np.savez_compressed(out, heights=H, x0=np.float32(-half), y0=np.float32(-half), cell=np.float32(cell))
    print("wrote", out, Path(out).stat().st_size, "bytes")
    return H


if __name__ == "__main__":
    H = main(Path(sys.argv[1]) / "wheeledlab_assets" / "data" / "Terrains" / "huge_compact.usd")
    # SURVEY 8c spot heights (decoded independently there): top surface z at (x, y)
    def at(x, y):
        return H[int(round((y + 20.5) / 0.1)), int(round((x + 20.5) / 0.1))]
    for (x, y, z) in [(0, 0, 0.2), (-2, 1, 0.2), (5.3, -7.7, 0.38109), (-12.2, 3.3, 0.47669), (19.9, 19.9, 0.2)]:
        print(f"z({x},{y}) = {at(x, y):.5f}   expected {z}")
