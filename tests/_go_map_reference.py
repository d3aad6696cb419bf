"""The exact reference of tests/_reduce_cases.py read as Go's map itself: what lh_reduce_sparse_host is held to.

processHistograms (metrics.go:336-418) iterates a map[int16]*uint64.  A map merged from several sets can hold a key
whose counts summed to 0 ((k, 2^64-1) plus (k, 1)); it is an entry like any other.  It takes part in the sort, so p <= 0
with a total above 0 picks the smallest key present (float64(0)/float64(total) >= p), and decompress(key) * 0 is NaN for
a key at +-Inf (precision <= 46), which makes the sum NaN.  Counts and running counts wrap at 2^64 as Go's uint64 do.
The snapshot's dense buckets cannot hold such keys, which is why rc.Reference drops them."""
import math

import numpy as np

import _reduce_cases as rc


class GoMapReference(rc.Reference):
    """rc.Reference (sum, sum of |terms|, nnz and the export arrays over the non-empty buckets) with the value order,
    running counts and sum of the Go map, zero-count keys included."""

    def __init__(self, hist: dict, table: np.ndarray, name: str = ""):
        super().__init__(hist, table, name)
        items = sorted(((float(table[k & 0xFFFF]), k, c) for k, c in hist.items()), key=lambda t: (t[0], t[1]))
        self.order = [k for _, k, _ in items]
        self.count %= 2 ** 64
        self.cums = []
        ratios = []
        sofar = 0
        for _, _, c in items:
            sofar = (sofar + c) % 2 ** 64
            self.cums.append(sofar)
            if self.count:
                ratios.append(float(sofar) / float(self.count))
            else:                                                  # Go: x / 0.0 is +Inf, 0 / 0.0 is NaN
                ratios.append(math.inf if sofar else math.nan)
        self.ratios = np.array(ratios, dtype=np.float64)
        if any(math.isinf(v) and c == 0 for v, _, c in items):
            self.sum = math.nan                                    # Inf * float64(0)
