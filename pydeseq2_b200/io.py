"""Count-matrix ingestion (SURVEY.md §8 f-4): CSV -> the (samples, genes) int64 matrix of the hot path, parsed by native host
threads straight into a page-locked buffer, so that the upload that follows runs at the full PCIe rate and nothing is copied or
converted on the way.  The reference loads the same files with ``pandas.read_csv(path, index_col=0).T``
(``examples/plot_pandas_io_example.py:57-66``) and converts to integers at construction (``dds.py:245-249``).
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib


@dataclass
class CountsTable:
    counts: np.ndarray   # (samples, genes) int64, C-contiguous; page-locked when a context was given
    samples: list        # row labels of `counts`
    genes: list          # column labels of `counts`

    def to_frame(self):
        """The ``counts_df`` of the reference's examples (samples x genes)."""
        import pandas as pd

        return pd.DataFrame(self.counts, index=self.samples, columns=self.genes)


def read_counts_csv(path, genes_in_rows: bool = True, sep: str = ",", ctx=None, threads: int = 0) -> CountsTable:
    """Parse a count table.  ``genes_in_rows`` (the layout of the reference's shipped datasets and of most count files: one line
    per gene, one column per sample): the table is transposed while it is parsed.  ``ctx`` (a ``_lib.Context``, e.g.
    ``B200Inference()._ops.ctx``): the matrix lands in page-locked memory.  Raises ``ValueError`` for a field that is not a
    non-negative integer (the reference rejects such tables in ``utils.test_valid_counts``, utils.py:100-133)."""
    lib = _lib.load()
    bpath = str(path).encode()
    bsep = sep.encode()[:1]
    n_rows, n_cols, nbytes = C.c_int64(), C.c_int64(), C.c_size_t()
    if lib.pdq_csv_scan(bpath, bsep, C.byref(n_rows), C.byref(n_cols), C.byref(nbytes)) != 0:
        raise OSError(f"cannot read {path!r}")
    R, K = n_rows.value, n_cols.value
    shape = (K, R) if genes_in_rows else (R, K)
    out = ctx.pinned_empty(shape, np.int64) if ctx is not None else np.empty(shape, dtype=np.int64)
    labels = C.create_string_buffer(nbytes.value + 16)
    bad_r, bad_c = C.c_int64(-1), C.c_int64(-1)
    rc = lib.pdq_csv_read_counts(bpath, bsep, 1 if genes_in_rows else 0, _lib.as_i64p(out), shape[1], R, K, labels, len(labels),
                                 int(threads), C.byref(bad_r), C.byref(bad_c))
    if rc != 0:
        if bad_r.value >= 0:
            raise ValueError(f"{path}: data row {bad_r.value}, column {bad_c.value} is not a non-negative integer read count")
        raise ValueError(f"{path}: malformed count table")
    raw = labels.raw
    cols, _, rest = raw.partition(b"\0")
    rows = rest.split(b"\0", 1)[0]
    col_names = cols.decode().split("\n")[:-1] if cols else []
    row_names = rows.decode().split("\n")[:-1] if rows else []
    samples, genes = (col_names, row_names) if genes_in_rows else (row_names, col_names)
    return CountsTable(out, samples, genes)


def to_pinned(counts, ctx) -> np.ndarray:
    """(samples, genes) counts from a DataFrame / array as a page-locked int64 matrix (one conversion pass)."""
    a = np.asarray(counts.values if hasattr(counts, "values") else counts)
    out = ctx.pinned_empty(a.shape, np.int64)
    np.copyto(out, a, casting="unsafe")
    return out
