"""TEST INFRASTRUCTURE: small end-to-end run of regk_dns_answer for compute-sanitizer (memcheck / racecheck / synccheck):
a mixed snapshot resolved from the host and the device, random query mixes with malformed messages from host and
device memory, host and device outputs, UDP and TCP, and the bad-offset refusal.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_dns_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import torch
from registrar_b200 import _native
import dns_util as du
import test_dns as t

ctx = _native.Context(0)
rng = random.Random(4)
nodes = t.random_snapshot(rng, n_dom=40)
nodes += [(b"/big", t.service(b"_h", b"_tcp", 80, 30))] + [(b"/big/i%d" % i, t.host(b"rr_host", b"10.0.0.1", None, [1, 2]))
                                                             for i in range(3000)]
zone = du.Zone(nodes)
msgs = t.random_queries(rng, nodes, zone, 2000) + [du.query(b"_h._tcp.big", du.T_SRV), du.query(b"big")]
mb, mo = du.pack(msgs)
dm, do = torch.from_numpy(mb).cuda(), torch.from_numpy(mo).cuda()
for snap in (t.host_snapshot(nodes), t.device_snapshot(nodes)):
    ctx.resolve(snap, 30, 60)
    for tcp in (False, True):
        ctx.answer_dns(mb, mo, 1232, tcp)
        ctx.answer_dns(dm, do, 1232, tcp, device=True)
bad = do.clone()
bad[5] = dm.numel() + 9
try:
    ctx.answer_dns(dm, bad)
    raise AssertionError("bad offsets were accepted")
except _native.RegkError as e:
    assert e.code == 1
torch.cuda.synchronize()
ctx.close()
print("sanitize_dns_run ok")
