"""TEST INFRASTRUCTURE: small end-to-end run of regk_read_results for compute-sanitizer (memcheck / racecheck /
synccheck), the companion of tests/sanitize_children_run.py: host and device streams of create, delete and setData
replies singly and in multi transactions (rolled back ones included), notifications and pings, a start inside the
stream, a stream that ends at its device allocation's last byte, and refusals.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_results_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from registrar_b200 import _native
from registrar_b200.batch import RecordBatch
import results_util as su
import test_read_results as t

ctx = _native.Context(0)
paths, pays = t.run(ctx, RecordBatch.from_records(t.fleet_records(1500, 20, seed=3)))
base = t.model_of(paths, pays, skip=set(range(0, len(paths), 7)))
for op in (t.ZK_CREATE, t.ZK_DELETE, t.ZK_SETDATA):
    for g in (0, 5):
        fb, fo, _ = ctx.jute_requests(op, xid_base=2 ** 31 - 10, group=g)
        s = su.Server(t.copy_model(base), t.SESSION).replies(fb, fo, extra={0: su.ping(), 4: su.notification(b"/q" * 30)},
                                                            header_err={2: -4})
        fr = su.Framing(op, paths, [len(p) for p in pays], 2 ** 31 - 10, g, su.NONODE if op == t.ZK_DELETE else 0)
        t.check(ctx, s, fr, t.RES_BATCH)
        t.check(ctx, b"\x01" * 7 + s, fr, t.RES_BATCH, start=7)
        exact = torch.from_numpy(np.frombuffer(s, np.uint8).copy()).cuda()         # no slack behind the last byte
        assert ctx.read_results(exact, t.RES_BATCH).n_failed == ctx.read_results(np.frombuffer(s, np.uint8), t.RES_BATCH).n_failed
        for bad in (s[:-40], s[:300] + b"\0\0\0\x05" + s[300:]):
            try:
                ctx.read_results(np.frombuffer(bad, np.uint8), t.RES_BATCH)
                raise AssertionError("a broken stream was accepted")
            except _native.RegkError as e:
                assert e.code == 1
torch.cuda.synchronize()
ctx.close()
print("sanitize_results_run ok")
