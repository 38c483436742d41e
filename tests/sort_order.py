"""The order of vexb_sort / vexb_sort_merge restated in numpy: the permutation a stable sort applies.

Ascending is numpy's stable argsort, which already treats -0.0 and +0.0 as equal and puts every NaN last.  Descending is
a stable argsort of the negated dense rank of the keys (-0.0 canonicalised to +0.0, NaNs ranked above +inf and equal to
each other), which needs no negation of the keys themselves and so no overflow at integer minima."""
import numpy as np


def permutation(keys: np.ndarray, descending: bool = False) -> np.ndarray:
    keys = np.asarray(keys)
    if not descending:
        return np.argsort(keys, kind="stable")
    canon = keys
    if keys.dtype.kind == "f":
        canon = np.where(keys == 0, np.zeros((), keys.dtype), keys)           # -0.0 -> +0.0; NaN stays NaN
    _, rank = np.unique(canon, return_inverse=True)                            # np.unique collapses NaNs into one, last
    return np.argsort(-rank.reshape(-1).astype(np.int64), kind="stable")


def sorted_bits(keys: np.ndarray, vals=None, descending: bool = False):
    """(keys, vals) as the stable sort leaves them."""
    p = permutation(keys, descending)
    return np.asarray(keys)[p], (None if vals is None else np.asarray(vals)[p])


def bits(a: np.ndarray) -> np.ndarray:
    """The array as unsigned integers of its width, so comparisons see -0.0 and NaN payloads."""
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])
