"""TEST INFRASTRUCTURE: small end-to-end run of regk_resolve for compute-sanitizer (memcheck / racecheck / synccheck):
a mixed snapshot from the host and the device, with host and device outputs, a service with many children, the
duplicate-path and bad-offset refusals.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_resolve_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import torch
from registrar_b200 import _native
from registrar_b200.batch import Snapshot
import test_resolve as t

ctx = _native.Context(0)
nodes = t.random_snapshot(random.Random(4), n_dom=60)
nodes += [(b"/big", t.service(b"_h", b"_tcp", 80, 30))] + [(b"/big/i%d" % i, t.host(b"rr_host", b"10.0.0.1", None, [1, 2]))
                                                             for i in range(3000)]
for snap in (t.host_snapshot(nodes), t.device_snapshot(nodes)):
    ctx.resolve(snap, 30, 60)
    ctx.resolve(snap, 30, 60, device=True)
for bad in (nodes + [nodes[3]], ):
    try:
        ctx.resolve(t.device_snapshot(bad), 30, 60)
        raise AssertionError("a duplicate path was accepted")
    except _native.RegkError as e:
        assert e.code == 1
d = t.device_snapshot(nodes)
off = d.path_off.clone()
off[5] = d.path_bytes.numel() + 9
try:
    ctx.resolve(Snapshot(d.path_bytes, off, d.json_bytes, d.json_off), 30, 60)
    raise AssertionError("bad offsets were accepted")
except _native.RegkError as e:
    assert e.code == 1
torch.cuda.synchronize()
ctx.close()
print("sanitize_resolve_run ok")
