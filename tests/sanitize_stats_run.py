"""TEST INFRASTRUCTURE: small end-to-end run of the exists framing, regk_read_stats and regk_reconcile_stats for
compute-sanitizer (memcheck / racecheck / synccheck), the companion of tests/sanitize_children_run.py: host and device
streams with notifications, pings and errors, both candidate kernels, a start inside the stream, a stream that ends at its
device allocation's last byte, the classification with and without a baseline, the repair frames, and refusals.  Run on
the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_stats_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import numpy as np
import torch
from registrar_b200 import _native, synth
import stats_util as su
import test_read_stats as t

ctx = _native.Context(0)
paths, pays = t.run(ctx, synth.generate("config3", n=3000, seed=21))
zk = t.registry(paths, pays, random.Random(4), same_length=True)
xid = 2 ** 31 - 10
fb = t.exists(ctx, paths, xid)
stream = su.replies(zk, fb, extra={0: su.ping(), 9: su.notification(b"/x" * 40)}, trailing=b"\0\0\0")
st = t.check(ctx, paths, stream, xid)
t.check(ctx, paths, b"\x01" * 7 + stream, xid, start=7)
exact = torch.from_numpy(np.frombuffer(stream[:-3], np.uint8).copy()).cuda()       # no slack behind the last byte
for shared in (0, 1):
    ctx.set_option("stats_cand_shared", shared)
    assert ctx.read_stats(exact).n_found == st.n_found
ctx.set_option("stats_cand_shared", 0)
for known in (None, st.mzxid + 1, torch.from_numpy(st.mzxid.copy()).cuda()):
    d = ctx.reconcile_stats(st, session=t.SESSION, zk_flags=1, known_mzxid=known)
    assert d.n_same + d.n_create + d.n_update + d.n_dup + d.n_replace == d.n
    t.repair_frames(ctx, groups=(0, 7))
for bad in (stream[:-40], stream[:500] + b"\0\0\0\x05" + stream[500:]):
    try:
        ctx.read_stats(np.frombuffer(bad, np.uint8))
        raise AssertionError("a broken stream was accepted")
    except _native.RegkError as e:
        assert e.code == 1
st = ctx.read_stats(np.frombuffer(su.replies(zk, fb, errors={5: -4}), np.uint8))
try:
    ctx.reconcile_stats(st, session=t.SESSION)
    raise AssertionError("an unknown node state was classed")
except _native.RegkError as e:
    assert e.code == 5
torch.cuda.synchronize()
ctx.close()
print("sanitize_stats_run ok")
