"""kvidx -- Python binding of libkvidx (the GPU-resident KV-block locality index).

The product is the CUDA library behind include/kvidx.h; this package only binds it
(ctypes) and mirrors the reference's host-side interface for the same path.
"""
from ._native import (Index, KvidxError, Config, Stats, EVENT_DTYPE, E, SCORE_ABSENT, LIB_PATH, SYMBOLS,  # noqa: F401
                      OK, ENOENT, ECUDA, ENOMEM, EINVAL, ENOSPC, ERANGE, EV_BLOCK_STORED, EV_BLOCK_REMOVED,
                      PAYLOAD_SKIP_UNKNOWN_TIER, PAYLOAD_STOP_AT_CLEARED, PAYLOAD_COUNTS,
                      load, fnv64a, podtier, host_alloc, host_free, pinned_array, snapshot_merge, pack_text)
