"""Reader of the Criteo Display Advertising TSV format (the Kaggle challenge's train.txt and the Terabyte day_* files).

Every line has 40 tab-separated columns: the label (0 or 1), 13 integer features and 26 categorical values of 8 hex
digits; any column but the label may be empty. Batches are what ``models.dlrm.DLRM.step`` takes:

* dense float32 [B, 13]: ``log(1 + max(v, 0))`` of a present value, 0 for a missing one;
* ids int64 [B, 26]: with ``per_field = num_features // 26`` keys per field, a missing value of field f is key
  ``f * per_field`` and a present value h is ``f * per_field + 1 + int(h, 16) % (per_field - 1)``;
* labels float32 [B].
"""
from __future__ import annotations

from typing import Iterator

import numpy as np
import torch

CRITEO_DENSE = 13
CRITEO_FIELDS = 26
CRITEO_COLUMNS = 1 + CRITEO_DENSE + CRITEO_FIELDS


def criteo_batches(path: str, batch_size: int, num_features: int) -> Iterator[tuple]:
    """Yields ``(dense, ids, labels)`` batches of ``batch_size`` lines of the file (the last batch may be shorter).
    A malformed line - a column count other than 40, a label other than 0 or 1, a non-numeric integer feature or a
    categorical value that is not hexadecimal - raises ``ValueError`` naming its line number (from 1)."""
    per_field = num_features // CRITEO_FIELDS
    if batch_size < 1:
        raise ValueError(f"batch_size must be >= 1, got {batch_size}")
    if per_field < 2:
        raise ValueError(f"num_features must give at least 2 keys per field (>= {2 * CRITEO_FIELDS}), got {num_features}")
    base = np.arange(CRITEO_FIELDS, dtype=np.int64) * per_field
    dense, ids, labels = [], [], []
    with open(path, "r", encoding="ascii", newline="") as fh:
        for n, line in enumerate(fh, 1):
            cols = line.rstrip("\r\n").split("\t")
            if len(cols) != CRITEO_COLUMNS:
                raise ValueError(f"{path}:{n}: expected {CRITEO_COLUMNS} tab-separated columns, got {len(cols)}")
            if cols[0] not in ("0", "1"):
                raise ValueError(f"{path}:{n}: the label must be 0 or 1, got {cols[0]!r}")
            try:
                d = [np.log1p(max(int(v), 0)) if v else 0.0 for v in cols[1:1 + CRITEO_DENSE]]
            except ValueError:
                raise ValueError(f"{path}:{n}: an integer feature is not an integer") from None
            try:
                c = [1 + int(v, 16) % (per_field - 1) if v else 0 for v in cols[1 + CRITEO_DENSE:]]
            except ValueError:
                raise ValueError(f"{path}:{n}: a categorical value is not hexadecimal") from None
            labels.append(float(cols[0]))
            dense.append(d)
            ids.append(c)
            if len(labels) == batch_size:
                yield _batch(dense, ids, labels, base)
                dense, ids, labels = [], [], []
    if labels:
        yield _batch(dense, ids, labels, base)


def _batch(dense, ids, labels, base):
    return (torch.from_numpy(np.asarray(dense, dtype=np.float32)),
            torch.from_numpy(np.asarray(ids, dtype=np.int64) + base),
            torch.from_numpy(np.asarray(labels, dtype=np.float32)))
