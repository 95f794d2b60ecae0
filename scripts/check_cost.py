"""What tsgpu_check_object costs against tsgpu_detransform over the same stored object: a 1 GiB Kafka segment with corpus-K record
payloads (tests/records_util.py) in 4 MiB chunks, host buffers (pinned), alternating in one process.  Objects: Zstd+AES written by
this library in speed and in dense mode, and Zstd+AES written by the oracle (libzstd level 3 + OpenSSL: what the Java plugin
wrote; its frames decode one CTA per frame).  The check runs without and with TSGPU_FLAG_VALIDATE_RECORDS.  Prints one JSON line:
  e2e        GiB/s of original bytes per call: median, min, max over the repeats, for detransform (to a pinned dst), check and
             check_records, and each check over detransform as a ratio of throughputs (> 1: the check is faster)
  kernel_ms  ms per GiB of original bytes of every kernel of one check_records call (per-kernel CUDA events of
             tsgpu_profile_report, in one separate profiled run)
  object_over_segment   transformed bytes per original byte: what crosses PCIe for the check
  gpu, power_limit_w    the card the numbers were taken on, read in the same call
Usage: python scripts/check_cost.py [--repeats 7] [--out FILE]"""
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
import numpy as np  # noqa: E402
import torch  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import binding, corpus  # noqa: E402
from oracle import oracle as ora  # noqa: E402
import records_util as R  # noqa: E402

MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
Z, A, D, VR = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VALIDATE_RECORDS


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
        raise SystemExit("check_cost.py measures on a GPU; none is visible")
    lib = binding.load()
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    seg = R.gen_segment(5, SEG - MIB, payload=corpus.gen_segment("K", 5, 64 * MIB, MIB), big=64 << 10)
    n = seg.size
    nch = (n + CS - 1) // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    k8, a8 = np.frombuffer(key, np.uint8), np.frombuffer(aad, np.uint8)
    dst = pinned(n + 64)
    osz = np.zeros(nch + 1, np.uint32)
    objects = {
        "ZA_speed": ctx.transform(Z | A, seg, CS, key, aad, ivs),
        "ZA_dense": ctx.transform(Z | D | A, seg, CS, key, aad, ivs),
        "ZA_libzstd": ora.transform_segment(Z | A, seg, CS, key, aad, ivs),
    }
    gib = n / (1 << 30)
    res = {"segment_bytes": n, "chunk_mib": CS // MIB, "corpus": "K payloads in Kafka record batches", "repeats": args.repeats,
           "e2e": {}, "kernel_ms": {}, "object_over_segment": {}}
    for mode, (obj_, sizes_) in objects.items():
        obj = pinned(obj_.size)
        obj[:] = obj_
        sizes = np.asarray(sizes_, np.uint32)
        cur = np.zeros(binding.CHECK_CURSOR_SIZE, np.uint8)
        o_crc, s_crc = binding.C.c_uint32(0), binding.C.c_uint32(0)

        def detransform():
            rc = lib.tsgpu_detransform(ctx.handle, Z | A, obj.ctypes.data, obj.size, sizes.ctypes.data, sizes.size,
                                       k8.ctypes.data, a8.ctypes.data, a8.size, dst.ctypes.data, dst.size, osz.ctypes.data)
            if rc:
                raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())

        def check(flags):
            cur[:] = 0
            rc = lib.tsgpu_check_object(ctx.handle, flags, obj.ctypes.data, obj.size, sizes.ctypes.data, sizes.size, CS, n,
                                        k8.ctypes.data, a8.ctypes.data, a8.size, cur.ctypes.data, 1, binding.C.addressof(o_crc),
                                        binding.C.addressof(s_crc))
            if rc:
                raise tsgpu.TsgpuError(rc, lib.tsgpu_last_error().decode())

        runs = {"detransform": detransform, "check": lambda: check(Z | A), "check_records": lambda: check(Z | A | VR)}
        e2e = {k: [] for k in runs}
        for rep in range(args.repeats + 2):
            for name, fn in runs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                dt = time.perf_counter() - t0
                if rep >= 2:
                    e2e[name].append(gib / dt)
        r = {k: stats(v, 2) for k, v in e2e.items()}
        for k in ("check", "check_records"):
            r[k + "_over_detransform"] = round(r[k]["median"] / r["detransform"]["median"], 3)
        res["e2e"][mode] = r
        res["object_over_segment"][mode] = round(obj.size / n, 4)
        ctx.profile_enable(True)
        check(Z | A | VR)
        rep_ = ctx.profile_report()
        ctx.profile_enable(False)
        ks = {k: round(v["ms"] / gib, 3) for k, v in rep_.items()}
        ks["all_kernels"] = round(sum(v["ms"] for v in rep_.values()) / gib, 3)
        res["kernel_ms"][mode] = ks
    ctx.close()
    res["gpu"], res["power_limit_w"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
