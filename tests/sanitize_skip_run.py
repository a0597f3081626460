"""TEST INFRASTRUCTURE: small end-to-end run of skip mode (REGK_SKIP_BAD) for compute-sanitizer (memcheck /
racecheck / synccheck), the companion of tests/sanitize_run.py: dirty batches through the fence, compaction,
second run and offset expansion on each host route, every result compared with the oracle.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_skip_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
from registrar_b200 import _native, synth
from registrar_b200.batch import FLAG_NO_JSON, FLAG_NO_PATH, RecordBatch
from oracle import oracle
from skip_util import fence_bits

ctx = _native.Context(0)


def dirty(n, alias=False, empty_labels=False):
    base = synth.generate("config3", n=n, start=5)
    recs = [base.record(i) for i in range(n)]
    for i in sorted({0, 127, 128, n // 3, n - 1}):
        recs[i] = dict(recs[i], address=b"" if i % 2 else b"1.2.3.\"4")
    for i in sorted({1, n // 2}):
        recs[i] = dict(recs[i], domain=b"a/b." + recs[i]["domain"], hostname=b"")
    if empty_labels:
        for i in (2, n // 4):
            recs[i] = dict(recs[i], domain=b"x..y." + recs[i]["domain"])
    return RecordBatch.from_records(recs, types=base.types, alias=alias)


def check(got, b, flags=0):
    bits = fence_bits(b, flags)
    want = oracle.register_batch(b.take(np.nonzero(bits == 0)[0]), flags_extra=flags)
    before = np.zeros(b.n + 1, np.int64)
    np.cumsum(bits == 0, out=before[1:])
    assert np.array_equal(got.skipped, np.nonzero(bits)[0])
    assert np.array_equal(got.path_bytes, want.path_bytes) and np.array_equal(got.json_bytes, want.json_bytes)
    assert np.array_equal(np.asarray(got.path_off, np.uint64), want.path_off[before])
    assert np.array_equal(np.asarray(got.json_off, np.uint64), want.json_off[before])


b = dirty(700)
check(ctx.register_batch(b, skip_bad=True), b)
b = dirty(700, alias=True)
check(ctx.register_batch(b, skip_bad=True), b)
b = dirty(900, empty_labels=True)                                    # exact-offset redo inside the second run
check(ctx.register_batch(b, skip_bad=True), b)
b = dirty(600)
check(ctx.register_batch(b, payloads=False, skip_bad=True), b, FLAG_NO_JSON)
check(ctx.register_batch(b, paths=False, skip_bad=True), b, FLAG_NO_PATH)
ctx.set_option("force_generic", 1); check(ctx.register_batch(b, skip_bad=True), b); ctx.set_option("force_generic", 0)
ctx.set_option("offsets32", 1); check(ctx.register_batch(b, skip_bad=True), b); ctx.set_option("offsets32", 0)
ctx.set_option("chunk_records", 512)                                 # pipelined host route
b = dirty(3000)
check(ctx.register_batch(b, skip_bad=True), b)
ctx.set_option("chunk_records", 262144)
ctx.set_option("async", 1)                                           # a dirty and a clean host batch in flight
b1, b2 = dirty(2000), synth.generate("config2", n=1500, start=9)
t1 = ctx.submit(b1, skip_bad=True); t2 = ctx.submit(b2, skip_bad=True)
check(ctx.collect(t1, copy=True), b1)
check(ctx.collect(t2, copy=True), b2)
ctx.set_option("async", 0)
print("sanitize_skip_run ok")
