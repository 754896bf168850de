"""The block rule of the subtiled passes (regress_out's column sums, the Pearson residual variance, combat's moments):
blocks are whole subtiles, bounded by the partials' scratch and, for a dense X, by settings.chunk_size."""
import pytest

from scanpy_b200 import _ops
from scanpy_b200._compat import settings

T = _ops.SUBTILE_ROWS


# (scratch bytes, bytes per subtile, chunk_size, subtiles per block for a CSR X, for a dense X)
@pytest.mark.parametrize("scratch, subtile, chunk, csr, dense", [
    (8000, 800, 50_000, 10, 10),     # the scratch bounds both
    (8000, 800, 3 * T + 5, 10, 3),   # chunk_size bounds a dense X, rounded down to whole subtiles
    (8000, 800, 10, 10, 1),          # a chunk_size below one subtile still gives one
    (100, 800, 50_000, 1, 1),        # a scratch below one subtile's partials still gives one
    (1 << 28, 24_000, T, 11184, 1),
])
def test_blocks_are_whole_subtiles_within_scratch_and_chunk(monkeypatch, scratch, subtile, chunk, csr, dense):
    monkeypatch.setattr(settings, "chunk_size", chunk)
    assert _ops.subtile_block_rows(False, scratch, subtile) == csr * T
    assert _ops.subtile_block_rows(True, scratch, subtile) == dense * T
