"""`sc.experimental` (src/scanpy/experimental/__init__.py): the analytic Pearson residuals route, in `pp`."""
from . import pp  # noqa: F401
