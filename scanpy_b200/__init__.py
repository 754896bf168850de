"""scanpy_b200 — H100-native (sm_90a) `pp.pca -> pp.neighbors -> tl.leiden` with scanpy's signatures.

    import scanpy_b200 as sb
    sb.pp.pca(adata); sb.pp.neighbors(adata); sb.tl.leiden(adata)

writes `.obsm['X_pca']`, `.varm['PCs']`, `.uns['pca']`, `.obsp['distances'|'connectivities']`,
`.uns['neighbors']`, `.obs['leiden']`, `.uns['leiden']` exactly as scanpy does.  All arithmetic runs
in hand-written CUDA behind the C ABI in include/scanpy_b200.h; there is no CPU fallback.
"""
from . import experimental, get, metrics, pp, tl  # noqa: F401
from ._compat import MiniAnnData, settings  # noqa: F401
from ._io import ZarrCSR, read_zarr_backed  # noqa: F401
from .transformer import B200KNNTransformer, B200PCA  # noqa: F401

__version__ = "0.1.0"
