"""Inputs shared by the emulator and the GPU tests of the frame executor."""
import numpy as np


def executor_shapes():
    """Inputs whose libzstd frames drive the frame executor's pointer-jumping steps into every branch (DESIGN.md §4.3)."""
    rng = np.random.default_rng(77)
    out = {}
    out["zeros"] = np.zeros(400000, dtype=np.uint8)                                   # one giant match, offset 1 (periodic source)
    blk = rng.integers(0, 256, 5000, dtype=np.uint8)
    out["period5000"] = np.tile(blk, 70)                                              # giant matches, offset 5000 >= the CTA (rounds)
    blk2 = rng.integers(0, 256, 700, dtype=np.uint8)
    out["period700"] = np.tile(blk2, 400)                                             # giant matches, offset < the CTA
    rec = rng.integers(97, 123, 120, dtype=np.uint8)                                  # records that differ in one byte: ~1 literal + ~100
    recs = np.tile(rec, 3000).reshape(3000, 120).copy()                               # bytes of match per sequence, chained back record
    recs[np.arange(3000), rng.integers(0, 120, 3000)] = rng.integers(65, 91, 3000, dtype=np.uint8)   # by record: a step of 1024
    out["records"] = recs.reshape(-1)                                                 # sequences spans > 32 KiB (cut) and chains deep
    mix = np.concatenate([out["records"][:100000], np.zeros(70000, dtype=np.uint8), rng.integers(0, 256, 30000, dtype=np.uint8),
                          out["period700"][:90000], out["records"][5000:90000]])
    out["mixed"] = mix
    return out
