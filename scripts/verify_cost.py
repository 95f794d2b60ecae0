"""What TSGPU_FLAG_VERIFY costs: host-buffer tsgpu_transform of a 1 GiB K segment in 4 MiB chunks (pinned buffers), Z|A in
speed and in dense mode, flag off and on alternating in one process.  Prints one JSON line:
  e2e        GiB/s (original bytes per second of the whole call) per mode and flag: median, min, max over the repeats
  added_ms_per_gib   a separate profiled run on one work slot (kernels back to back, so each CUDA-event span is the kernel's
                     own time): ms per GiB of every kernel the flag adds, and their sum
  gpu, power_limit_w the card the numbers were taken on
Usage: python scripts/verify_cost.py [--repeats 7] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402

MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
Z, A, D, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY
MODES = {"speed": Z | A, "dense": Z | D | A}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return q[0], float(q[1])
    except Exception:                                    # noqa: BLE001 — the name still comes from torch
        return torch.cuda.get_device_name(0), None


def pinned(n):
    return torch.empty(n, dtype=torch.uint8).pin_memory().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("verify_cost.py measures on a GPU; none is visible")
    nch = SEG // CS
    src = pinned(SEG)
    src[:] = np.resize(corpus.gen_segment("K", 0, 16 * CS, CS), SEG)      # 16 distinct chunks, repeated
    key, aad, ivs = corpus.fixed_key_material(nch)
    dst = pinned(int(tsgpu.binding.load().tsgpu_transform_bound(Z | A, SEG, CS)) + 64)

    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    runs = {(m, v): [] for m in MODES for v in (False, True)}
    for rep in range(args.repeats + 2):                                    # two rounds of warm-up
        for m, flags in MODES.items():
            for v in (False, True):
                t0 = time.perf_counter()
                ctx.transform(flags | (V if v else 0), src, CS, key, aad, ivs, dst=dst)
                dt = time.perf_counter() - t0
                if rep >= 2:
                    runs[(m, v)].append(SEG / dt / (1 << 30))
    ctx.close()

    os.environ["TSGPU_SLOTS"] = "1"
    pctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    added = {}
    for m, flags in MODES.items():
        rep_ = {}
        for v in (False, True):
            pctx.transform(flags | (V if v else 0), src, CS, key, aad, ivs, dst=dst)     # warm-up
            pctx.profile_enable(True)
            pctx.transform(flags | (V if v else 0), src, CS, key, aad, ivs, dst=dst)
            rep_[v] = pctx.profile_report()
            pctx.profile_enable(False)
        new = {k: round(e["ms"] * (1 << 30) / SEG, 3) for k, e in rep_[True].items() if k not in rep_[False]}
        added[m] = dict(new, total=round(sum(new.values()), 3))
    pctx.close()

    name, plim = gpu_info()
    res = {"segment_gib": SEG / (1 << 30), "chunk_mib": CS // MIB, "corpus": "K", "repeats": args.repeats, "gpu": name,
           "power_limit_w": plim, "e2e": {}, "added_ms_per_gib": added}
    for m in MODES:
        row = {}
        for v in (False, True):
            x = runs[(m, v)]
            row["on" if v else "off"] = {"median": round(statistics.median(x), 2), "min": round(min(x), 2), "max": round(max(x), 2)}
        row["median_cost_pct"] = round(100.0 * (1 - row["on"]["median"] / row["off"]["median"]), 1)
        res["e2e"][m] = row
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
