"""Write tests/golden/pbmc68k_regress.npz from a checkout of the reference (scverse/scanpy).

It holds what the reference's `test_regress_out_reproducible` (tests/test_preprocessing.py:472-488) needs besides the
raw X, which pbmc68k_raw_seurat_hvg.npz already has (its input is `raw[:200, :200]`):
* obs/n_counts, obs/percent_mito and obs/bulk_labels/codes of src/scanpy/datasets/10x_pbmc68k_reduced.zarr.zip;
* the goldens tests/_data/regress_test_small.npy (keys n_counts, percent_mito) and regress_test_small_cat.npy
  (key bulk_labels), 200 x 200 float64.

Usage:  python tests/golden/make_regress.py <scanpy checkout>   (writes next to this file)
"""
from __future__ import annotations

import sys
import zipfile
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_goldens import read_zarr_array  # noqa: E402

OUT = Path(__file__).resolve().parent


def main() -> None:
    ref = Path(sys.argv[1])
    z = zipfile.ZipFile(ref / "src/scanpy/datasets/10x_pbmc68k_reduced.zarr.zip")
    out = {
        "n_counts": read_zarr_array(z, "obs/n_counts"),
        "percent_mito": read_zarr_array(z, "obs/percent_mito"),
        "bulk_labels_codes": read_zarr_array(z, "obs/bulk_labels/codes"),
        "regress_test_small": np.load(ref / "tests/_data/regress_test_small.npy"),
        "regress_test_small_cat": np.load(ref / "tests/_data/regress_test_small_cat.npy"),
    }
    np.savez_compressed(OUT / "pbmc68k_regress.npz", **out)
    for k, v in out.items():
        print(k, v.shape, v.dtype)


if __name__ == "__main__":
    main()
