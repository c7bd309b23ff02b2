"""vega_b200 — H100-native (sm_90a) shuffle + aggregation engine behind vega's RDD operator API.

The product is vega_b200/libvega_b200.so (C ABI in include/vega_b200.h, CUDA kernels in
vega_b200/csrc/).  This package is the host-side mirror of the reference's operator
interface for the path (rdd.py) plus the one-process-per-GPU exchange (dist.py).
Importing works without a GPU (so the C ABI can be inspected); computing does not.
"""
from ._lib import (LIB_PATH, SYMBOLS, VegaB200Error, lib)  # noqa: F401
from .rdd import (AggregateRdd, CoGroupedRdd, CombinedRdd, Context, Grouped, JoinedRdd, PairRdd, Rdd, RepartitionedRdd, RepShuffle, SemiJoinedRdd,  # noqa: F401
                  Shuffle, ShuffledRdd,
                  BytesKeys, StrAggregateRdd, StrCoGroupedRdd, StrCombinedRdd, StrKeys, StrPairRdd, StrRdd, StrShuffle, StrShuffledRdd, StrSortedRdd, slice_starts)

__all__ = ["Context", "PairRdd", "CoGroupedRdd", "CombinedRdd", "AggregateRdd", "Rdd", "RepartitionedRdd", "RepShuffle", "SemiJoinedRdd", "Shuffle", "ShuffledRdd", "JoinedRdd", "Grouped", "slice_starts",
           "BytesKeys", "StrAggregateRdd", "StrCoGroupedRdd", "StrCombinedRdd", "StrKeys", "StrPairRdd", "StrRdd", "StrShuffle", "StrShuffledRdd", "StrSortedRdd", "VegaB200Error", "lib", "LIB_PATH", "SYMBOLS"]
