"""Run by tests/test_simt_reframe.py in a subprocess (argv[1] = the library to load: the ASan build, or the plain emulator build
with poisoned scratch or another lane order): TSGPU_FLAG_REFRAME over objects from 1 byte to several batches in chunks from 1 byte
to 4 KiB, one and two chunks per slot batch, in one call and in windows, from libzstd and from this library's speed and dense
frames, with and without checksum and with skippable frames after them; the dense candidates on libzstd's frames.  The seal kernel's block walk, its in-place move of the
skippable frames and the pick kernel's copy are checked for overruns and for what they write; damaged sources must fail, never
overrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
from oracle import oracle as ora  # noqa: E402
import part_crc_util as U  # noqa: E402
import reframe_util as F  # noqa: E402
import rewrite_util as W  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
Z, A, D, CK, RF = F.Z, F.A, F.D, F.CK, F.RF

for max_batch in (1, 2):
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=max_batch, lib_path=lib)
    for cs, n in ((1, 40), (257, 3000), (4096, 4096 * 3 + 17)):
        src = corpus.gen_segment("K", cs, n, cs)
        nch = (n + cs - 1) // cs
        chunks = F.chunks_of(src, cs)
        nk, na, nivs = W.new_key_material(nch)
        dense = {ck: W.frames(Z, *c.transform(Z | D | ck, src, cs)) for ck in (0, CK)}
        sources = [("oracle",) + tuple(ora.transform_segment(Z, src, cs))]
        sources.append(("skippable",) + F.with_skippable(*sources[0][1:], every=1))
        for wf in (Z, Z | CK):
            o, s = c.transform(wf, src, cs)
            sources.append((wf, o.copy(), s))
        for name, obj, sizes in sources:
            old = W.frames(Z, obj, sizes)
            # the dense candidates on the oracle's frames only: the compressor has sweeps of its own
            for tf in (Z | CK | RF, Z | CK | A | RF) + ((Z | D | RF, Z | D | CK | A | RF) if name == "oracle" else ()):
                want = F.expected(tf, old, chunks, dense[tf & CK])
                for win in ((None, 3) if tf == Z | CK | RF else (None,)):
                    new, nsz, parts, crc3 = W.rewrite_windows(c, Z, obj, sizes, cs, n, tf, 1000, win, None, b"", nk, na, nivs)
                    assert W.frames(tf, new, nsz, nk, na) == want, (cs, name, tf, win)
                    assert crc3 == (U.crc32c(obj), U.crc32c(new), U.crc32c(src)), (cs, name, tf, win)
            # a damaged frame fails as the source's invalid frame, whatever REFRAME would have written
            bad = obj.copy()
            at = int(sum(sizes[:nch // 2]))
            bad[at + min(sizes[nch // 2] - 1, 6)] ^= 0x5A
            try:
                W.rewrite_windows(c, Z, bad, sizes, cs, n, Z | D | CK | RF, 1000, None, None, b"", nk, na, nivs)
            except tsgpu.TsgpuError as e:
                assert e.code in (tsgpu.binding.E_CORRUPT, tsgpu.binding.E_VERIFY), str(e)
            else:
                raise AssertionError("a damaged %s source was rewritten (cs %d)" % (name, cs))
    c.close()
print("reframe sweep ok")
