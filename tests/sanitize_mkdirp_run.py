"""TEST INFRASTRUCTURE: small end-to-end run of regk_mkdirp_dirs / regk_mkdirp_requests for compute-sanitizer
(memcheck / racecheck / synccheck), the companion of tests/sanitize_run.py: host, alias (empty and control-byte labels),
fleet, skip-mode and tight-table batches, every set and its frames compared with the restatement in mkdirp_util.
Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_mkdirp_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from registrar_b200 import _native, synth
from registrar_b200.batch import RecordBatch
from oracle import oracle
from mkdirp_util import mkdirp_frames, mkdirp_set

ctx = _native.Context(0)


def check(paths):
    dirs, first, invalid = mkdirp_set(paths)
    ds = ctx.mkdirp_dirs()
    assert ds.dirs() == dirs and ds.dir_rec.tolist() == first and ds.invalid.tolist() == invalid
    fb, fo, _ = ctx.mkdirp_requests(xid_base=2 ** 31 - 5)
    assert fb.tobytes() == mkdirp_frames(dirs, 2 ** 31 - 5, 0)
    return ds


def run(batch, **kw):
    got = ctx.register_batch(batch, **kw)
    return [got.path(i) for i in range(got.n) if got.skipped is None or i not in set(got.skipped.tolist())]


check(run(synth.generate("config3", n=3000, start=5)))
doms = [b"a..b", b"a.", b"", b"x\x01.y", b"m." * 70 + b"n", b"c.b.a", b"a.b"] * 50
check(run(RecordBatch.from_records([{"domain": d, "hostname": b"h", "type": b"host", "address": b"1.1.1.1"} for d in doms],
                                   alias=True)))
recs = [{"domain": b"svc%d.example.com" % (i % 9), "hostname": b"h" * (1 + i % 13), "type": b"host", "address": b"1.1.1.1"}
        for i in range(2000)]
check(run(RecordBatch.from_records(recs)))
base = synth.generate("config3", n=1000, start=9)
dirty = [base.record(i) for i in range(base.n)]
for i in (0, 500, 999):
    dirty[i] = dict(dirty[i], address=b"")
check(run(RecordBatch.from_records(dirty, types=base.types), skip_bad=True))
ctx.set_option("mkdirp_tight_table", 1)
check(run(synth.generate("config3", n=2000, start=11)))
ctx.set_option("mkdirp_tight_table", 0)
ctx.close()
print("sanitize_mkdirp_run ok")
