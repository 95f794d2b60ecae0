"""Where the speed-mode compressor's cycles go, per 8 KiB block: one 1 GiB K segment in 4 MiB chunks through
transform_device (flags Zstd + AES, as bench.py's default line) with a library built with -DZB_TUNE_PHASES=1:

    scripts/ab_variants.sh phases "-DZB_TUNE_PHASES=1"      # -> ab/libtsgpu_phases.so
    python scripts/enc_phases.py [--lib ab/libtsgpu_phases.so] [--out FILE]

Every warp stamps clock64() at its block's phase boundaries (ZbPhases in zstd_enc_blk.cuh).  Prints one JSON line: per
phase the median and p90 SM cycles per block and the phase's share of all cycles, plus the medians of the block's
sequence, literal and literal-symbol counts and the card the numbers were taken on.  A phase a block skips (raw literals,
no sequences) counts 0 cycles there; its work is charged to the next phase the block records."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402

MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
ZB = 8192
PHASES = ["stage", "parse", "huffman_table", "literals", "fse_tables", "seq_stream", "lookback", "copy"]
REC = np.dtype([("t", "<u8", 9), ("nseq", "<u4"), ("nlit", "<u4"), ("nsym", "<u4"), ("pad", "<u4")])


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return q[0], float(q[1])
    except Exception:                                    # noqa: BLE001 — the name still comes from torch
        return torch.cuda.get_device_name(0), None


def main():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(root, "ab", "libtsgpu_phases.so"))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("enc_phases.py measures on a GPU; none is visible")
    lib = tsgpu.binding.load(args.lib)
    if not hasattr(lib, "tsgpu_zb_phases"):
        raise SystemExit("%s was not built with -DZB_TUNE_PHASES=1" % args.lib)
    lib.tsgpu_zb_phases.argtypes = [C.c_void_p, C.c_uint64]

    nch = SEG // CS
    flags = tsgpu.FLAG_ZSTD | tsgpu.FLAG_AES
    key, aad, ivs = corpus.fixed_key_material(nch)
    dev = torch.device("cuda", 0)
    d_src = torch.from_numpy(corpus.gen_segment("K", 0, SEG, CS)).to(dev)
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=nch, devices=[0], lib_path=args.lib)
    stride = ctx.slot_stride(flags, CS)
    d_slots = torch.empty(nch * stride, dtype=torch.uint8, device=dev)
    d_sizes = torch.zeros(nch, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream().cuda_stream
    for _ in range(3):                                   # the last call's records are read
        ctx.transform_device(flags, d_src.data_ptr(), SEG, CS, key, aad, ivs, d_slots.data_ptr(), stride,
                             d_sizes.data_ptr(), stream)
    torch.cuda.synchronize()
    nblk = SEG // ZB
    rec = np.zeros(nblk, dtype=REC)
    if lib.tsgpu_zb_phases(rec.ctypes.data, rec.nbytes) != 0:
        raise SystemExit("tsgpu_zb_phases: %s" % lib.tsgpu_last_error().decode())
    ratio = SEG / float(d_sizes.cpu().numpy().astype(np.int64).sum())
    ctx.close()

    t = rec["t"].astype(np.int64)
    if (t[:, 0] == 0).any() or (t[:, 8] == 0).any():
        raise SystemExit("some blocks left no record: %d" % int(((t[:, 0] == 0) | (t[:, 8] == 0)).sum()))
    for k in range(1, 9):                                # a skipped phase takes the previous stamp: 0 cycles
        t[:, k] = np.where(t[:, k] == 0, t[:, k - 1], t[:, k])
    d = np.diff(t, axis=1)
    total = float(d.sum())
    name, plim = gpu_info()
    res = {"gpu": name, "power_limit_w": plim, "segment_gib": SEG / (1 << 30), "chunk_mib": CS // MIB, "corpus": "K",
           "blocks": nblk, "compression_ratio": round(ratio, 4),
           "block_cycles": {"median": int(np.median(d.sum(1))), "p90": int(np.percentile(d.sum(1), 90))},
           "phases": {p: {"median": int(np.median(d[:, i])), "p90": int(np.percentile(d[:, i], 90)),
                          "share_pct": round(100.0 * d[:, i].sum() / total, 1)} for i, p in enumerate(PHASES)},
           "median_nseq": int(np.median(rec["nseq"])), "median_nlit": int(np.median(rec["nlit"])),
           "median_nsym": int(np.median(rec["nsym"]))}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
