"""What TSGPU_FLAG_ZSTD_CHECKSUM costs, flag off and on alternating in one process, on a 1 GiB K segment in 4 MiB chunks.
Prints one JSON line:
  device     ms per 1 GiB device-resident tsgpu_transform_device (Z, CUDA events around the call), speed and dense mode:
             median, min, max over the repeats, and on/off as a ratio of throughputs (1.0 = free)
  e2e        GiB/s of the host-buffer tsgpu_transform (Z|A, pinned buffers), speed and dense mode, same statistics
  fetch_ms   ms per 16 MiB window (4 chunks, host-buffer tsgpu_detransform of Z|A frames this library wrote with and without
             the checksum), speed and dense frames
  gpu, power_limit_w  the card the numbers were taken on
Usage: python scripts/checksum_cost.py [--repeats 7] [--out FILE]"""
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
WIN = 4
Z, A, D, C = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_ZSTD_CHECKSUM
MODES = {"speed": 0, "dense": D}


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
        raise SystemExit("checksum_cost.py measures on a GPU; none is visible")
    nch = SEG // CS
    src = pinned(SEG)
    src[:] = np.resize(corpus.gen_segment("K", 0, 16 * CS, CS), SEG)      # 16 distinct chunks, repeated
    key, aad, ivs = corpus.fixed_key_material(nch)
    res = {"segment_gib": SEG / (1 << 30), "chunk_mib": CS // MIB, "corpus": "K", "repeats": args.repeats}

    # device-resident: the kernels alone
    dctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=nch)
    d_src = torch.from_numpy(src).cuda()
    stride = dctx.slot_stride(Z, CS)
    slots = torch.empty(nch * stride, dtype=torch.uint8, device="cuda")
    sizes = torch.empty(nch, dtype=torch.int32, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev = {(m, c): [] for m in MODES for c in (False, True)}
    for rep in range(args.repeats + 2):
        for m, mf in MODES.items():
            for c in (False, True):
                e0.record()
                dctx.transform_device(Z | mf | (C if c else 0), d_src.data_ptr(), SEG, CS, None, b"", None, slots.data_ptr(),
                                      stride, sizes.data_ptr())
                e1.record()
                e1.synchronize()
                if rep >= 2:
                    dev[(m, c)].append(e0.elapsed_time(e1))
    del slots, sizes, d_src
    dctx.close()
    res["device"] = {}
    for m in MODES:
        off, on = stats(dev[(m, False)]), stats(dev[(m, True)])
        res["device"][m] = {"off_ms": off, "on_ms": on, "on_over_off_throughput": round(off["median"] / on["median"], 4)}

    # host-buffer, end to end; then 16 MiB fetch windows of the frames it wrote
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    dst = pinned(int(tsgpu.binding.load().tsgpu_transform_bound(Z | A, SEG, CS)) + 64)
    e2e = {(m, c): [] for m in MODES for c in (False, True)}
    objs = {}
    for rep in range(args.repeats + 2):
        for m, mf in MODES.items():
            for c in (False, True):
                t0 = time.perf_counter()
                out, tsz = ctx.transform(Z | A | mf | (C if c else 0), src, CS, key, aad, ivs, dst=dst)
                dt = time.perf_counter() - t0
                if rep >= 2:
                    e2e[(m, c)].append(SEG / dt / (1 << 30))
                if rep == 0:
                    k0 = 100
                    a = sum(tsz[:k0])
                    objs[(m, c)] = (out[a:a + sum(tsz[k0:k0 + WIN])].copy(), tsz[k0:k0 + WIN])
    res["e2e"] = {}
    for m in MODES:
        off, on = stats(e2e[(m, False)], 2), stats(e2e[(m, True)], 2)
        res["e2e"][m] = {"off_gib_s": off, "on_gib_s": on, "on_over_off": round(on["median"] / off["median"], 4)}
    wdst = pinned(WIN * CS)
    fetch = {k: [] for k in objs}
    for rep in range(5 * args.repeats + 5):
        for k, (win, tsz) in objs.items():
            t0 = time.perf_counter()
            ctx.detransform(Z | A, win, tsz, WIN * CS, key, aad, dst=wdst)
            dt = time.perf_counter() - t0
            if rep >= 5:
                fetch[k].append(dt * 1e3)
    ctx.close()
    res["fetch_ms"] = {}
    for m in MODES:
        off, on = stats(fetch[(m, False)]), stats(fetch[(m, True)])
        res["fetch_ms"][m] = {"off": off, "on": on, "added_ms": round(on["median"] - off["median"], 3)}

    res["gpu"], res["power_limit_w"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
