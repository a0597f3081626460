"""TEST INFRASTRUCTURE: small end-to-end run of regk_dns_answer with REGK_DNS_PTR for compute-sanitizer (memcheck /
racecheck / synccheck): a snapshot with shared addresses resolved from the host and the device, the reverse index
built and reused, reverse and forward query mixes from host and device memory, host and device outputs, UDP and TCP,
one address shared by 3 000 hosts, and an empty index.  Run on the GPU box:
    compute-sanitizer --tool memcheck python tests/sanitize_dns_ptr_run.py"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import random
import torch
from registrar_b200 import _native
import dns_ptr_util as pu
import dns_util as du
import test_dns as t
import test_dns_ptr as tp

ctx = _native.Context(0)
rng = random.Random(4)
nodes = tp.shared_snapshot(rng, 30)
nodes += [(b"/big/i%d" % i, t.host(b"host", b"10.0.0.9")) for i in range(3000)]
zone = du.Zone(nodes)
msgs = t.random_queries(rng, nodes, zone, 1000) + tp.reverse_queries(rng, tp.addrs_of(zone), 1000)
msgs.append(du.query(pu.reverse_name(b"10.0.0.9"), pu.T_PTR, opt=(4096, 0, 0)))
mb, mo = du.pack(msgs)
dm, do = torch.from_numpy(mb).cuda(), torch.from_numpy(mo).cuda()
for snap in (t.host_snapshot(nodes), t.device_snapshot(nodes)):
    ctx.resolve(snap, 30, 60)
    for tcp in (False, True):
        ctx.answer_dns(mb, mo, 1232, tcp, ptr=True)
        ctx.answer_dns(dm, do, 1232, tcp, device=True, ptr=True)
        ctx.answer_dns(mb, mo, 1232, tcp)
ctx.resolve(t.host_snapshot([(b"/us/x", t.service())]), 30, 60)
ctx.answer_dns(mb, mo, 1232, False, ptr=True)
torch.cuda.synchronize()
ctx.close()
print("sanitize_dns_ptr_run ok")
