"""Small host-side pieces of scanpy's runtime that the three hot-path functions lean on.

* `MiniAnnData` — a duck-typed stand-in for `anndata.AnnData` (anndata is not installed in the build
  image).  The public functions only use `.X .obs .var .obsm .varm .obsp .uns .n_obs .n_vars
  .shape .is_view .copy()`, `adata[:, mask]` and the in-place subsetting the filters call
  (`_inplace_subset_obs` / `_inplace_subset_var`), so a real AnnData works unchanged.
* `settings` — the two constants the path reads (`N_PCS`, `n_jobs`; src/scanpy/_settings/__init__.py:83,132)
  plus verbosity-free logging with the reference's message texts (src/scanpy/logging.py:100-131).
* `accepts_legacy_random_state` — the `random_state=` <-> `rng=` shim of
  src/scanpy/_utils/random.py:182-208: a bare call or `random_state=` records
  `params['random_state']` in `.uns`, an explicit `rng=` does not.
"""
from __future__ import annotations

import logging
import time
import warnings
from functools import wraps
from types import SimpleNamespace

import numpy as np
import pandas as pd
from scipy import sparse

logger = logging.getLogger("scanpy_b200")

settings = SimpleNamespace(N_PCS=50, n_jobs=4, chunk_size=50_000)  # anndata's default chunk_size for chunked_X is 6000; the device path prefers larger row chunks


def log_start(msg: str) -> float:
    logger.info(msg)
    return time.perf_counter()


def log_done(start: float, deep: str = "") -> None:
    logger.info("    finished (%.3fs)%s", time.perf_counter() - start, (" " + deep) if deep else "")


def warn(msg: str, category=UserWarning) -> None:
    warnings.warn(msg, category, stacklevel=3)


class LegacyRng:
    """Marker: the caller used the legacy `random_state` form (value kept in `.arg`)."""

    def __init__(self, arg):
        self.arg = arg

    def generator(self) -> np.random.Generator:
        return np.random.default_rng(self.arg if self.arg is not None else None)


def accepts_legacy_random_state(default_seed):
    """`f(..., rng=None)` gains a `random_state=` keyword; neither given -> legacy default seed."""

    def deco(fn):
        @wraps(fn)
        def wrapper(*args, random_state="__unset__", rng=None, **kw):
            if rng is not None and random_state != "__unset__":
                raise TypeError("Specify at most one of `rng` and `random_state`.")
            if rng is None:
                rng = LegacyRng(default_seed if random_state == "__unset__" else random_state)
            return fn(*args, rng=rng, **kw)

        return wrapper

    return deco


def seed_from_rng(rng) -> int:
    """Integer seed for the CUDA kernels from either form."""
    if isinstance(rng, LegacyRng):
        if isinstance(rng.arg, (int, np.integer)):
            return int(rng.arg) & 0xFFFFFFFFFFFFFFFF
        return int(np.random.default_rng(None if rng.arg is None else rng.arg).integers(0, 2**31 - 1))
    return int(np.random.default_rng(rng).integers(0, 2**31 - 1))


def meta_random_state(rng) -> dict:
    return dict(random_state=rng.arg) if isinstance(rng, LegacyRng) else {}


class _AxisArrays(dict):
    pass


class MiniAnnData:
    """Minimal AnnData look-alike: enough surface for pca/neighbors/leiden and their tests."""

    def __init__(self, X=None, obs=None, var=None, obsm=None, varm=None, obsp=None, uns=None, layers=None):
        self.X = X
        self.layers = dict(layers or {})
        n_obs, n_vars = self.shape if X is not None or self.layers else (len(obs), len(var))
        self.obs = obs if obs is not None else pd.DataFrame(index=pd.RangeIndex(n_obs).astype(str))
        self.var = var if var is not None else pd.DataFrame(index=pd.RangeIndex(n_vars).astype(str))
        self.obsm = _AxisArrays(obsm or {})
        self.varm = _AxisArrays(varm or {})
        self.obsp = _AxisArrays(obsp or {})
        self.uns = dict(uns or {})
        self.is_view = False
        self.isbacked = False

    @property
    def shape(self):
        """X's shape; with X None (a result made of layers only, like `get.aggregate`'s) the first layer's, else
        (len(obs), len(var))."""
        if self.X is not None:
            return self.X.shape
        if self.layers:
            return next(iter(self.layers.values())).shape
        return (len(self.obs), len(self.var))

    @property
    def n_obs(self):
        return self.shape[0]

    @property
    def n_vars(self):
        return self.shape[1]

    @property
    def T(self):
        """The transpose: X and layers transposed, obs / var and obsm / varm swapped (obsp and uns are not carried)."""
        return MiniAnnData(None if self.X is None else self.X.T, self.var, self.obs, dict(self.varm), dict(self.obsm),
                           layers={k: v.T for k, v in self.layers.items()})

    def copy(self):
        import copy

        new = MiniAnnData(None if self.X is None else self.X.copy(), self.obs.copy(), self.var.copy(),
                          {k: v.copy() for k, v in self.obsm.items()}, {k: v.copy() for k, v in self.varm.items()},
                          {k: v.copy() for k, v in self.obsp.items()}, copy.deepcopy(self.uns))
        new.layers = {k: v.copy() for k, v in self.layers.items()}
        return new

    def _inplace_subset_obs(self, mask):
        """Keep the cells selected by `mask` (boolean or integer index): X, obs, obsm rows, obsp on both axes, layers."""
        idx = np.asarray(mask)
        self.X = self.X[idx]
        self.obs = self.obs.iloc[idx]
        self.obsm = _AxisArrays({k: v.iloc[idx] if hasattr(v, "iloc") else v[idx] for k, v in self.obsm.items()})
        self.obsp = _AxisArrays({k: v[idx][:, idx] for k, v in self.obsp.items()})
        self.layers = {k: v[idx] for k, v in self.layers.items()}

    def _inplace_subset_var(self, mask):
        """Keep the genes selected by `mask` (boolean or integer index): X, var, varm rows, layers."""
        idx = np.asarray(mask)
        self.X = self.X[:, idx]
        self.var = self.var.iloc[idx]
        self.varm = _AxisArrays({k: v.iloc[idx] if hasattr(v, "iloc") else v[idx] for k, v in self.varm.items()})
        self.layers = {k: v[:, idx] for k, v in self.layers.items()}

    def __getitem__(self, idx):
        if not (isinstance(idx, tuple) and len(idx) == 2 and isinstance(idx[0], slice) and idx[0] == slice(None)):
            raise NotImplementedError("MiniAnnData only supports adata[:, var_mask]")
        mask = np.asarray(idx[1])
        x = self.X[:, mask]
        sub = MiniAnnData(x, self.obs, self.var.loc[mask] if mask.dtype == bool else self.var.iloc[mask])
        sub.is_view = True
        return sub


def is_anndata_like(obj) -> bool:
    return all(hasattr(obj, a) for a in ("X", "obs", "var", "obsm", "varm", "obsp", "uns"))


def get_arr(adata, *, use_raw: bool = False, layer=None, obsm=None, obsp=None):
    """`_get_arr(adata, use_raw=..., layer=..., obsm=..., obsp=...)` along the cells (src/scanpy/get/get.py:545-570)."""
    if not isinstance(use_raw, bool):
        raise TypeError(f"use_raw expected to be bool, was {type(use_raw)}.")
    picked = [k for k, v in (("use_raw", use_raw), ("layer", layer), ("obsm", obsm), ("obsp", obsp))
              if v is not None and v is not False]
    if len(picked) > 1:
        valid = [f"`{k}`" for k in picked]
        valid[-1] = f"or {valid[-1]}"
        raise ValueError(f"Only one of {', '.join(valid)} can be specified.")
    if use_raw:
        return adata.raw.X
    if layer is not None:
        return adata.layers[layer]
    if obsm is not None:
        return adata.obsm[obsm]
    if obsp is not None:
        return adata.obsp[obsp]
    return adata.X


def as_csr_f32(x):
    """Input matrix -> scipy CSR with float32 data (float64 is down-cast: the kernels compute in fp32
    storage / fp64 accumulation; dense input is converted)."""
    if sparse.issparse(x):
        x = x.tocsr()
    else:
        x = sparse.csr_matrix(np.asarray(x))
    if x.dtype != np.float32:
        x = x.astype(np.float32)
    if not x.has_canonical_format:
        x = x.copy()
        x.sum_duplicates()
    return x
