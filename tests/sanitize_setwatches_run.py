"""TEST INFRASTRUCTURE: small end-to-end run of the watched heartbeat across a reconnect for compute-sanitizer
(memcheck / racecheck / synccheck), the companion of tests/sanitize_events_run.py: a watched round 0 read through
read_events, an unread re-check, SetWatches frames at the default, the minimum and a one-frame max_frame on the host and
the device, the server's answer read back through read_events, and a refused -8 reply.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_setwatches_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch
from registrar_b200 import _native
import setwatches_util as sw
import test_setwatches as t

ctx = _native.Context(0)
paths, pays = t.batch(ctx, n=3000, seed=21)
zk = t.session_model(paths, pays, missing=(7,))
t.arm(ctx, zk, paths)
zk.set_data(paths[12], b"x")
ctx.read_events(np.frombuffer(zk.take_events(t.SESSION), np.uint8))
ctx.events_requests(t.ZK_EXISTS, xid_base=70)
zk.drop_connection(t.SESSION)
lmax = max(len(p) for p in paths)
for mf in (32 + 2 * (4 + lmax), 2 ** 31 - 1):
    ctx.setwatches_requests(max_frame=mf)
    ctx.setwatches_requests(max_frame=mf, device=True)
sg = ctx.setwatches_requests()
s = zk.serve_setwatches(sg.frames.tobytes(), t.SESSION)
g = ctx.read_events(torch.from_numpy(np.frombuffer(s, np.uint8).copy()).cuda())
assert g.n_replies == sg.n_frames
try:
    ctx.read_events(np.frombuffer(sw.reply(1, err=-4), np.uint8))
    raise AssertionError("a SetWatches reply with an err was accepted")
except _native.RegkError as e:
    assert e.code == 1
torch.cuda.synchronize()
ctx.close()
print("sanitize_setwatches_run ok")
