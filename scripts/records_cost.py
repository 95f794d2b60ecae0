"""What TSGPU_FLAG_VALIDATE_RECORDS costs, flag off and on alternating in one process, on 1 GiB generated Kafka segments (K
payloads) in 4 MiB chunks, with small (1 KiB) and large (256 KiB) record batches.  Prints one JSON line:
  e2e        GiB/s of the host-buffer tsgpu_transform (Z|A, pinned buffers, speed mode): median, min, max over the repeats,
             and on/off as a ratio of throughputs (1.0 = free)
  kernel_ms  ms per GiB of each record kernel, their total, and all kernels of the call (per-kernel CUDA events of
             tsgpu_profile_report, in one separate profiled run)
  gpu, power_limit_w  the card the numbers were taken on
Usage: python scripts/records_cost.py [--repeats 7] [--out FILE]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
import records_util as R  # noqa: E402

MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
Z, A, VR = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_VALIDATE_RECORDS
SHAPES = {"1KiB": dict(small=1024, big=1025, legacy=0.0), "256KiB": dict(small=256 * 1024, big=256 * 1024 + 1, legacy=0.0)}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return q[0], float(q[1])
    except Exception:                                    # noqa: BLE001 — the name still comes from torch
        return torch.cuda.get_device_name(0), None


def pinned(n):
    return torch.empty(n, dtype=torch.uint8).pin_memory().numpy()


def stats(x, nd=3):
    return {"median": round(statistics.median(x), nd), "min": round(min(x), nd), "max": round(max(x), nd)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("records_cost.py measures on a GPU; none is visible")
    payload = corpus.gen_segment("K", 0, 64 * MIB, MIB)
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    res = {"segment_gib": SEG / (1 << 30), "chunk_mib": CS // MIB, "corpus": "K", "repeats": args.repeats, "e2e": {}, "kernel_ms": {}}
    for shape, opts in SHAPES.items():
        seg = R.gen_segment(0, SEG, payload=payload, **opts)                    # ends at the first entry end past 1 GiB
        src = pinned(seg.size)
        src[:] = seg
        nch = (src.size + CS - 1) // CS
        key, aad, ivs = corpus.fixed_key_material(nch)
        dst = pinned(int(tsgpu.binding.load().tsgpu_transform_bound(Z | A, src.size, CS)) + 64)
        e2e = {False: [], True: []}
        for rep in range(args.repeats + 2):
            for on in (False, True):
                t0 = time.perf_counter()
                ctx.transform(Z | A | (VR if on else 0), src, CS, key, aad, ivs, dst=dst)
                dt = time.perf_counter() - t0
                if rep >= 2:
                    e2e[on].append(src.size / dt / (1 << 30))
        off, on = stats(e2e[False], 2), stats(e2e[True], 2)
        res["e2e"][shape] = {"off_gib_s": off, "on_gib_s": on, "on_over_off": round(on["median"] / off["median"], 4),
                             "entries": int(R.starts(seg).size)}
        ctx.profile_enable(True)
        ctx.transform(Z | A | VR, src, CS, key, aad, ivs, dst=dst)
        rep_ = ctx.profile_report()
        ctx.profile_enable(False)
        gib = src.size / (1 << 30)
        ks = {k: round(v["ms"] / gib, 3) for k, v in rep_.items() if k.startswith("rec_")}
        ks["total"] = round(sum(ks.values()), 3)
        ks["all_kernels"] = round(sum(v["ms"] for v in rep_.values()) / gib, 3)
        res["kernel_ms"][shape] = ks
    ctx.close()
    res["gpu"], res["power_limit_w"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
