"""`sc.get` functions on the device: `aggregate`.

Reference: src/scanpy/get/_aggregated.py:242-404 (the `layer` / `obsm` / `varm` / `axis` API).  The grouping labels
are combined on the host (`combine_categories`); the per-group statistics run in CUDA (`_aggregate.group_stats`,
csrc/aggregate.cu).  Output dtypes are the reference's for each input kind:
* `sum`: int64 for an integer sparse X, float64 otherwise (a dense X goes through a float64 indicator product);
* `count_nonzero`: int64 for a sparse X, float64 for a dense one;
* `mean`, `var`: float64;
* `median`: float32 for a dense float32 X (np.median keeps it), float64 otherwise (a sparse X's medians fill a float64
  array; np.median of integers is float64).  Values are computed in the data's type, as there: the mean of the two
  middle float32 values is rounded to float32 before it is stored.
`mean` alone is Σx / n, as in `Aggregate.mean`; with `var` it is the mean of the same pass (`Aggregate.mean_var`), so a
group whose rows are all masked out has mean NaN in the first case and 0 in the second, as there.

Not implemented: `acc=` and `anndata.acc` references, graph (obsp / varp) aggregation, dask arrays, and input other
than an AnnData (or this package's `MiniAnnData`).
"""
from __future__ import annotations

from itertools import product

import numpy as np
import pandas as pd
from scipy import sparse

from ._compat import MiniAnnData, is_anndata_like, warn

AGG_FUNCS = ("count_nonzero", "sum", "median", "mean", "var")  # `get_literal_vals(AggType)`, in its order


def _literal_vals():
    return dict.fromkeys(AGG_FUNCS).keys()


def _is_ref(obj) -> bool:
    return type(obj).__module__.startswith("anndata.acc")


def resolve_axis(axis):
    """`_resolve_axis`: 0 / "obs" or 1 / "var" -> (index, name)."""
    if axis in {0, "obs"}:
        return 0, "obs"
    if axis in {1, "var"}:
        return 1, "var"
    raise ValueError(f"`axis` must be either 0, 1, 'obs', or 'var', was {axis!r}")


def combine_categories(label_df: pd.DataFrame) -> tuple[pd.Categorical, pd.DataFrame]:
    """One categorical over the combinations of the columns' levels -> (the rows' combined categorical, the label frame
    of its categories).  Every column's unused levels are dropped first; combinations are named "_".join of their
    levels in `itertools.product` order (the last column varies fastest), and those no row has are dropped.  A row with
    a missing label in any column has no category."""
    cols = list(label_df.columns)
    cats = [pd.Categorical(label_df[c]).remove_unused_categories() for c in cols]
    levels = [c.categories for c in cats]
    sizes = [len(lv) for lv in levels]
    grid = np.indices(sizes).reshape(len(cols), -1)
    names = pd.Index(["_".join(map(str, combo)) for combo in product(*levels)])
    labels = pd.DataFrame({c: pd.Categorical.from_codes(grid[i], levels[i]) for i, c in enumerate(cols)}, index=names)
    codes = np.zeros(len(label_df), dtype=np.int64)
    missing = np.zeros(len(label_df), dtype=bool)
    stride = 1
    for cat, size in zip(reversed(cats), reversed(sizes), strict=True):
        codes += cat.codes.astype(np.int64) * stride
        missing |= cat.codes < 0
        stride *= size
    codes[missing] = -1
    result = pd.Categorical.from_codes(codes, categories=names).remove_unused_categories()
    return result, labels.loc[result.categories]


def check_mask(adata, mask, dim: str):
    """`_check_mask` for a boolean mask: a column name of `adata.obs` / `adata.var` or an array."""
    if mask is None:
        return None
    if _is_ref(mask):
        raise NotImplementedError("aggregate in scanpy_b200 does not implement `anndata.acc` references for `mask`")
    if isinstance(mask, str):
        try:
            mask_array = np.asarray(getattr(adata, dim)[mask])
        except KeyError:
            raise ValueError(f"Did not find `adata.{dim}[{mask!r}]`. ") from None
    else:
        if len(mask) != adata.shape[0 if dim == "obs" else 1]:
            raise ValueError("The shape of the mask do not match the data.")
        mask_array = mask
    if not pd.api.types.is_bool_dtype(mask_array.dtype):
        raise ValueError("Mask array must be boolean.")
    return mask_array


def get_data(adata, dim: str, *, layer=None, obsm=None, varm=None):
    """`_get_arr(adata, dim=dim, layer=..., obsm=..., varm=...)`: the matrix with the grouped axis along the rows."""
    picked = [(k, v) for k, v in (("layer", layer), ("obsm", obsm), ("varm", varm)) if v is not None and v is not False]
    if not picked:
        return adata.X.T if dim == "var" else adata.X
    if len(picked) > 1:
        valid = [f"`{k}`" for k, _ in picked]
        valid[-1] = f"or {valid[-1]}"
        raise ValueError(f"Only one of {', '.join(valid)} can be specified.")
    k, v = picked[0]
    if k == "layer":
        return adata.layers[v].T if dim == "var" else adata.layers[v]
    if k == "obsm":
        if dim == "var":
            raise ValueError("`obsm` cannot be used when `dim` is `var`")
        return adata.obsm[v]
    if dim == "obs":
        raise ValueError("`varm` cannot be used when `dim` is `obs`")
    return adata.varm[v]


def check_funcs(func) -> set:
    funcs = set([func] if isinstance(func, str) else func)
    if unknown := funcs - _literal_vals():
        raise ValueError(f"func {unknown} is not one of {_literal_vals()}")
    return funcs


def _check_data(data):
    mod = type(data).__module__
    if mod.startswith("dask") or hasattr(data, "dask"):
        raise NotImplementedError("aggregate in scanpy_b200 does not implement dask arrays")
    if isinstance(data, pd.DataFrame):
        return data.values
    if isinstance(data, np.ndarray) or (sparse.issparse(data) and data.format in ("csr", "csc")):
        return data
    raise NotImplementedError(f"Data type {type(data)} not supported for aggregation")


def finish(stats: dict, funcs: set, categories: pd.Index, *, sparse_input: bool, integer: bool, dof: int) -> dict:
    """The result layers from the device statistics, in the reference's order, dtypes and NaN rules."""
    counts = stats["counts"]
    result = {}
    if "sum" in funcs:
        result["sum"] = stats["sum"].astype(np.int64) if sparse_input and integer else stats["sum"]
    if "mean" in funcs and "var" not in funcs:
        result["mean"] = stats["sum"] / counts[:, None]
    if "count_nonzero" in funcs:
        result["count_nonzero"] = stats["nnz"] if sparse_input else stats["nnz"].astype(np.float64)
    if "var" in funcs:
        n = counts[:, None].astype(np.float64)
        var = np.divide(stats["m2"], n, out=np.zeros_like(stats["m2"]), where=n > 0)
        if dof != 0:
            denom = np.where(counts > dof, counts - dof, np.nan)
            which_nan = np.isnan(denom)
            if which_nan.any():
                warn(f"Group counts matches dof, resulting var for groups {categories[which_nan].to_list()} will be "
                     "nan", RuntimeWarning)
            var *= (counts / denom)[:, np.newaxis]
        result["var"] = var
        if "mean" in funcs:
            result["mean"] = stats["mean"]
    if "median" in funcs:
        med = stats["median"]
        result["median"] = med.astype(np.float64) if sparse_input else med
    return result


def aggregate(adata, by, func, *, acc=None, mask=None, dof: int = 1, axis=None, layer=None, obsm=None, varm=None):
    """Aggregate the data matrix by a categorical grouping (signature of `scanpy.get.aggregate`'s `layer` / `obsm` /
    `varm` / `axis` API).

    `by`: a column name of `adata.obs` (`adata.var` with `axis="var"` or `varm`) or a list of names, combined into one
    grouping.  `func`: one of, or an iterable of, "count_nonzero", "sum", "median", "mean", "var"; each becomes a layer
    of the result.  `mask`: a boolean array or a column name; masked-out observations count in no group.  `dof`: the
    degrees of freedom of "var".  Returns an AnnData (a `MiniAnnData` when anndata is not installed) with one row per
    group that occurs, `n_obs_aggregated` in its obs, and the result transposed for `axis="var"`."""
    from . import _aggregate

    if not is_anndata_like(adata):
        raise NotImplementedError("sc.get.aggregate is currently only implemented for AnnData input, "
                                  f"was passed {type(adata)}.")
    if acc is not None:
        raise NotImplementedError("aggregate in scanpy_b200 does not implement `acc=` (anndata.acc accessors, including "
                                  "graph aggregation over obsp / varp); use `layer`, `obsm` or `varm`")
    by = [by] if isinstance(by, str) else list(by)
    if any(_is_ref(b) for b in by):
        raise NotImplementedError("aggregate in scanpy_b200 does not implement `anndata.acc` references for `by`")
    if axis is not None:
        dim = resolve_axis(axis)[1]
    elif varm:
        dim = "var"
    else:
        dim = "obs"
    data = _check_data(get_data(adata, dim, layer=layer, obsm=obsm, varm=varm))
    dim_df = pd.DataFrame({ref: getattr(adata, dim)[ref] for ref in by})
    mask = check_mask(adata, mask, dim)
    categorical, label_df = combine_categories(dim_df)
    codes = np.asarray(categorical.codes, dtype=np.int32).copy()
    if mask is not None:
        codes[~np.asarray(mask, dtype=bool)] = -1
    n_groups = len(categorical.categories)
    counts = np.bincount(codes[codes >= 0], minlength=n_groups)
    label_df["n_obs_aggregated"] = pd.Series(counts, index=categorical.categories).reindex(label_df.index)
    funcs = check_funcs(func)
    sparse_input = sparse.issparse(data)
    integer = np.dtype(data.dtype).kind in "iu"
    stats = _aggregate.group_stats(data, codes, n_groups, moments=bool(funcs - {"median"}), median="median" in funcs)
    layers = finish(stats, funcs, categorical.categories, sparse_input=sparse_input, integer=integer, dof=dof)
    if obsm or varm:
        src = get_data(adata, dim, obsm=obsm, varm=varm)
        var = pd.DataFrame(index=src.columns if isinstance(src, pd.DataFrame) else
                           pd.RangeIndex(src.shape[1]).astype(str))
    else:
        var = getattr(adata, "var" if dim == "obs" else "obs")
    result = make_result(layers, label_df, var)
    return result if dim == "obs" else result.T


def make_result(layers: dict, obs: pd.DataFrame, var: pd.DataFrame):
    """An anndata.AnnData when anndata is installed, else a `MiniAnnData` with X None."""
    try:
        from anndata import AnnData
    except ImportError:
        return MiniAnnData(None, obs=obs, var=var, layers=layers)
    return AnnData(layers=layers, obs=obs, var=var)
