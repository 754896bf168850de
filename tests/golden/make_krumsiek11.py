"""Regenerate tests/golden/krumsiek11.npz from a checkout of the reference (scverse/scanpy).

The fixture is the numeric table of the reference's src/scanpy/datasets/krumsiek11.txt (640 cells x 11 genes).
`sc.datasets.krumsiek11()` reads that file with `first_column_names=True`: column 0 holds the observation names, and the
last `#` comment line before the table names the genes.  The reference's own filter_cells docstring
(src/scanpy/preprocessing/_simple.py:104-133) pins what the filters give on it: after `X[X < 0.3] = 0`,
`filter_cells(min_genes=0)` keeps 640 cells with `n_genes.min() == 1` and `min_genes=3` keeps 554.

Usage:  python tests/golden/make_krumsiek11.py <scanpy checkout>   (writes next to this file)
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

OUT = Path(__file__).resolve().parent


def write_krumsiek11(ref: Path) -> None:
    lines = (ref / "src/scanpy/datasets/krumsiek11.txt").read_text().splitlines()
    header = [ln for ln in lines if ln.startswith("#")][-1].lstrip("#").split()
    rows = [ln.split() for ln in lines if ln.strip() and not ln.startswith("#")]
    np.savez_compressed(OUT / "krumsiek11.npz", X=np.array([r[1:] for r in rows], dtype=np.float32),
                        obs_names=np.array([r[0] for r in rows]), var_names=np.array(header[1:]))
    print("krumsiek11", len(rows), "x", len(header) - 1)


if __name__ == "__main__":
    write_krumsiek11(Path(sys.argv[1]))
