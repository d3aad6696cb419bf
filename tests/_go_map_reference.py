"""The exact reference of tests/_reduce_cases.py read as Go's map itself: what lh_reduce_sparse_host is held to.

processHistograms (metrics.go:336-418) iterates a map[int16]*uint64.  A map merged from several sets can hold a key
whose counts summed to 0 ((k, 2^64-1) plus (k, 1)); it is an entry like any other.  It takes part in the sort, so p <= 0
with a total above 0 picks the smallest key present (float64(0)/float64(total) >= p), while with a total that wrapped to
0 its ratio is 0/0.0 = NaN and p <= 0 picks the first non-empty key.  decompress(key) * 0 is NaN for a key at +-Inf
(precision <= 46), which makes the sum NaN.  The snapshot's dense buckets cannot hold such keys, which is why
rc.Reference drops them; counts, running counts and the total wrap at 2^64 in both, as Go's uint64 do."""
import math

import numpy as np

import _reduce_cases as rc


class GoMapReference(rc.Reference):
    """rc.Reference (sum, sum of |terms|, nnz and the export arrays over the non-empty buckets) with the value order,
    running counts and sum of the Go map, zero-count keys included."""

    def __init__(self, hist: dict, table: np.ndarray, name: str = ""):
        super().__init__(hist, table, name)
        self._rank(hist.items())
        if any(math.isinf(float(table[k & 0xFFFF])) and c == 0 for k, c in hist.items()):
            self.sum = math.nan                                    # Inf * float64(0)
