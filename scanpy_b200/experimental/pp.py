"""`sc.experimental.pp` (src/scanpy/experimental/pp/__init__.py): analytic Pearson residuals on the device."""
from .._pearson import (highly_variable_genes, normalize_pearson_residuals, normalize_pearson_residuals_pca,
                        recipe_pearson_residuals)

__all__ = [
    "highly_variable_genes",
    "normalize_pearson_residuals",
    "normalize_pearson_residuals_pca",
    "recipe_pearson_residuals",
]
