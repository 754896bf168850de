"""Write tests/golden/harmony_pbmc68k.npz from a checkout of the reference (scverse/scanpy).

It runs the reference's Harmony (src/scanpy/preprocessing/_harmony/core.py, loaded on its own with stub
`scanpy.logging`, `scanpy._settings` and `scanpy._utils.random` modules; beyond them it needs only numpy, sklearn and
tqdm) on the in-tree pbmc68k `X_pca` (700 x 50, pbmc68k_reduced_graph.npz) with `bulk_labels`
(pbmc68k_regress.npz), in float64 with rng=0, and records for each case:
* `<case>/centers`: the KMeans `cluster_centers_` of its k-means start (a recording KMeans subclass patched in);
* `<case>/iters`: the number of clustering iterations of every outer iteration;
* `<case>/out`: `X_pca_harmony` on the cells `rows` (every fifth cell: a fault in the schedule moves every row, and the
  full 700 x 50 float64 outputs of four cases would not compress below 1 MB).
`params` holds each case's keyword arguments as JSON; `batch2_codes` is the reference test's second key,
`default_rng(0).choice(["A", "B", "C"], size=700)`, as codes into ["A", "B", "C"].

Usage:  python tests/golden/make_harmony.py <scanpy checkout>   (writes next to this file)
"""
from __future__ import annotations

import importlib.util
import json
import sys
import types
from pathlib import Path

import numpy as np
import pandas as pd

OUT = Path(__file__).resolve().parent
ROW_STEP = 5

CASES = {
    "harmony2": dict(keys=["bulk_labels"]),
    "harmony1": dict(keys=["bulk_labels"], flavor="harmony1"),
    "two_keys": dict(keys=["bulk_labels", "batch2"], theta=[2.0, 0.1]),
    "tau": dict(keys=["bulk_labels"], tau=5, n_clusters=50, sigma=0.15),
}
DEFAULTS = dict(theta=2.0, sigma=0.1, n_clusters=None, max_iter_harmony=10, max_iter_clustering=200,
                tol_harmony=1e-4, tol_clustering=1e-5, ridge_lambda=1.0, block_proportion=0.05, tau=0, alpha=0.2,
                batch_prune_threshold=1e-5, flavor="harmony2", rng=0)


def _load_core(ref: Path):
    def module(name, **attrs):
        m = types.ModuleType(name)
        m.__path__ = []
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    def legacy_random_state(rng, /, *, always_state=False):
        [bitgen] = np.random.default_rng(rng).bit_generator.spawn(1)
        return np.random.RandomState(bitgen)

    module("scanpy")
    module("scanpy.logging", info=lambda *a, **k: None)
    module("scanpy._settings", settings=types.SimpleNamespace(verbosity=0))
    module("scanpy._settings.verbosity", Verbosity=types.SimpleNamespace(info=1))
    module("scanpy._utils")
    module("scanpy._utils.random", _legacy_random_state=legacy_random_state)
    module("scanpy.preprocessing")
    module("scanpy.preprocessing._harmony")
    name = "scanpy.preprocessing._harmony.core"
    spec = importlib.util.spec_from_file_location(name, ref / "src/scanpy/preprocessing/_harmony/core.py")
    core = importlib.util.module_from_spec(spec)
    sys.modules[name] = core
    spec.loader.exec_module(core)
    return core


def main() -> None:
    ref = Path(sys.argv[1])
    core = _load_core(ref)
    record = {}

    class RecordingKMeans(core.KMeans):
        def fit(self, x, *args, **kwargs):
            out = super().fit(x, *args, **kwargs)
            record["centers"] = self.cluster_centers_.copy()
            return out

    calls = [0]
    convergent = core._is_convergent_clustering
    clustering = core._clustering

    def counting_convergent(*args, **kwargs):
        calls[0] += 1
        return convergent(*args, **kwargs)

    def counting_clustering(*args, **kwargs):
        calls[0] = 0
        out = clustering(*args, **kwargs)
        record["iters"].append(calls[0])
        return out

    core.KMeans = RecordingKMeans
    core._is_convergent_clustering = counting_convergent
    core._clustering = counting_clustering

    x = np.load(OUT / "pbmc68k_reduced_graph.npz")["X_pca"].astype(np.float64)
    bulk = np.load(OUT / "pbmc68k_regress.npz")["bulk_labels_codes"].astype(np.int64)
    batch2 = np.random.default_rng(0).choice(["A", "B", "C"], size=len(x))
    obs = pd.DataFrame({"bulk_labels": pd.Categorical.from_codes(bulk, [f"b{i}" for i in range(bulk.max() + 1)]),
                        "batch2": batch2})
    rows = np.arange(0, len(x), ROW_STEP)
    out = {"batch2_codes": np.searchsorted(["A", "B", "C"], batch2).astype(np.int8), "rows": rows}
    params = {}
    for case, spec in CASES.items():
        kw = {**DEFAULTS, **{k: v for k, v in spec.items() if k != "keys"}}
        params[case] = {**kw, "keys": spec["keys"]}
        flavor = kw.pop("flavor")
        record.clear()
        record["iters"] = []
        h = core.Harmony(obs, spec["keys"], stabilized_penalty=flavor == "harmony2",
                         dynamic_lambda=flavor == "harmony2", **kw)
        res = h.fit(x)
        out[f"{case}/centers"] = record["centers"]
        out[f"{case}/iters"] = np.array(record["iters"], dtype=np.int32)
        out[f"{case}/out"] = res[rows]
        print(case, record["centers"].shape, record["iters"], float(np.abs(res).max()))
    out["params"] = np.array(json.dumps(params))
    np.savez_compressed(OUT / "harmony_pbmc68k.npz", **out)


if __name__ == "__main__":
    main()
