"""TEST INFRASTRUCTURE: small end-to-end run of regk_jute_requests(REGK_ZK_GETDATA) and regk_read_replies for
compute-sanitizer (memcheck / racecheck / synccheck), the companion of tests/sanitize_reconcile_owned_run.py: host and
device streams with notifications, pings, errors, duplicate paths, data that embeds reply frames, a stream that ends at
its device allocation's last byte, a registry repaired in the model, and refusals.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_replies_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import numpy as np
import torch
from registrar_b200 import _native, synth
import replies_util as ru
import test_read_replies as t

ctx = _native.Context(0)
paths, pays = t.run(ctx, synth.generate("config3", n=3000, start=5))
fb = t.getdata(ctx, paths, 2 ** 31 - 10)
zk = t.model_of(paths, pays, skip=set(range(0, 3000, 7)))
stream = ru.replies(zk, fb, errors={5: -4}, extra={0: ru.ping(), 9: ru.notification(b"/x" * 40)}, trailing=b"\0\0\0")
t.check(ctx, paths, stream, 2 ** 31 - 10)
exact = torch.from_numpy(np.frombuffer(stream[:-3], np.uint8).copy()).cuda()       # no slack behind the last byte
assert ctx.read_replies(exact).n_found == ctx.read_replies(np.frombuffer(stream, np.uint8)).n_found
for k, p in enumerate(paths[:20]):
    if p in zk.nodes:
        zk.nodes[p].data = stream[100 * k:100 * k + 2000]
t.check(ctx, paths, ru.replies(zk, fb), 2 ** 31 - 10)
for bad in (stream[:-40], stream[:500] + b"\0\0\0\x05" + stream[500:]):
    try:
        ctx.read_replies(np.frombuffer(bad, np.uint8))
        raise AssertionError("a broken stream was accepted")
    except _native.RegkError as e:
        assert e.code == 1
paths, pays = t.run(ctx, synth.generate("config3", n=1500, seed=21))
zk, dirs = t._build_registry(paths, pays, random.Random(4))
fb = t.getdata(ctx, paths, 3)
rep = t.check(ctx, paths, ru.replies(zk, fb), 3)
ctx.reconcile_owned(rep, session=t.SESSION, zk_flags=1)
t._repair(ctx, zk)
torch.cuda.synchronize()
ctx.close()
print("sanitize_replies_run ok")
