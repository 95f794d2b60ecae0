"""e2e (host pinned buffers through tsgpu_transform) vs batch size — tuning probe."""
import sys, time
sys.path.insert(0, '.')
import numpy as np, torch
import tsgpu
from tsgpu import corpus
MIB = 1 << 20
seg, cs = 1024 * MIB, 4 * MIB
nch = seg // cs
kind = sys.argv[1] if len(sys.argv) > 1 else 'K'
src = corpus.gen_segment(kind, 0, seg, cs)
h_src = torch.empty(seg, dtype=torch.uint8).pin_memory(); h_src.numpy()[:] = src
key, aad, ivs = corpus.fixed_key_material(nch)
import os
for flags, slots, mb in ((3, 16, 4), (3, 16, 8), (3, 16, 2), (3, 16, 16), (7, 16, 4), (1, 16, 4), (2, 16, 4), (2, 16, 8)):
    if True:
        os.environ['TSGPU_SLOTS'] = str(slots)
        ctx = tsgpu.Context(max_chunk_bytes=cs, max_batch=mb)
        cap = int(ctx.lib.tsgpu_transform_bound(flags, seg, cs)) + 64
        h_dst = torch.empty(cap, dtype=torch.uint8).pin_memory(); d = h_dst.numpy()
        for _ in range(2): ctx.transform(flags, h_src.numpy(), cs, key, aad, ivs, dst=d)
        torch.cuda.synchronize(); t0 = time.perf_counter()
        for _ in range(4): out, sizes = ctx.transform(flags, h_src.numpy(), cs, key, aad, ivs, dst=d)
        torch.cuda.synchronize(); dt = (time.perf_counter() - t0) / 4
        print('flags', flags, 'slots', slots, 'batch', mb, 'e2e %.1f GiB/s' % (1.0 / dt), 'out MiB', sum(sizes) // MIB, flush=True)
        ctx.close(); del h_dst
# raw copy ceilings
d_buf = torch.empty(seg, dtype=torch.uint8, device='cuda')
torch.cuda.synchronize(); t0 = time.perf_counter()
for _ in range(3): d_buf.copy_(h_src, non_blocking=True)
torch.cuda.synchronize(); print('H2D 1 GiB pinned: %.1f GiB/s' % (3.0 / (time.perf_counter() - t0)))
h2 = torch.empty(seg, dtype=torch.uint8).pin_memory()
torch.cuda.synchronize(); t0 = time.perf_counter()
for _ in range(3): h2.copy_(d_buf, non_blocking=True)
torch.cuda.synchronize(); print('D2H 1 GiB pinned: %.1f GiB/s' % (3.0 / (time.perf_counter() - t0)))
