"""regk_walk_resolve on the GPU: after every refresh of registry-shaped random scripts (and between events and the
refresh, with removed nodes still in the snapshot), every output array and count against resolve_util.resolve of the
model's nodes and against a plain regk_resolve of the same snapshot on a second context, with full, n_fresh and
copied_bytes as walk_resolve_util predicts them; regk_dns_answer after it against regk_dns_answer after regk_resolve;
the regk_dns_answer gate; full = 1 at the start, after walk_start and for changed TTLs; reuse across an interleaved
regk_resolve and across a reconnect; a refused call that changes nothing; the fleet at 1 000 x 4 000, 1 % churn."""
import hashlib
import random

import numpy as np
import pytest

import dns_util as du
import resolve_util as rv
import walk_resolve_util as wr
import walk_setwatches_util as ws
import walk_watch_util as ww
from test_resolve import compare, raw_to_dict
from test_resolve_cpu import host, service

pytestmark = pytest.mark.gpu
DH, DS = 30, 60
SESSION = 7


@pytest.fixture(scope="module")
def ctxs(built):
    from registrar_b200 import _native
    a, b = _native.Context(0), _native.Context(0)
    yield a, b
    a.close()
    b.close()


def _dict(ans):
    return dict(q_kind=ans.q_kind, q_node=ans.q_node, sec_off=ans.sec_off, text=ans.text, node_cls=ans.node_cls,
                unresolved=ans.unresolved, n_answers=ans.n_answers, n_additional=ans.n_additional)


def same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


def walk_resolve(ctx, dh, ds, device):
    """-> (arrays as a dict, (full, n_fresh, copied_bytes, formatted_bytes), text_total)"""
    if device:
        out = ctx.walk_resolve(dh, ds, device=True)
        return raw_to_dict(ctx, out.answers), (int(out.full), int(out.n_fresh), int(out.copied_bytes),
                                               int(out.formatted_bytes)), int(out.answers.text_total)
    a = ctx.walk_resolve(dh, ds)
    return _dict(a), (a.full, a.n_fresh, a.copied_bytes, a.formatted_bytes), a.text_total


def plain(ctx2, walk, dh, ds):
    return _dict(ctx2.resolve(walk, dh, ds))


class Checker:
    """walk_resolve after each phase, against the restatement, a plain resolve and the predicted counters"""

    def __init__(self, ctx, ctx2, rng):
        self.ctx, self.ctx2, self.rng, self.copied, self.calls = ctx, ctx2, rng, 0, 0

    def __call__(self, d, phase, dh=DH, ds=DS):
        m = d.model
        full, fresh, copied = m.predict(dh, ds)
        got, counts, total = walk_resolve(self.ctx, dh, ds, self.rng.random() < 0.5)
        compare(got, rv.resolve(m.pairs(), dh, ds))
        same(got, plain(self.ctx2, self.ctx._walk, dh, ds))
        assert counts == (full, fresh, copied, total - copied), phase
        m.resolved(dh, ds)
        self.copied += copied
        self.calls += 1


@pytest.mark.parametrize("seed", range(8))
def test_random_registry_scripts(ctxs, seed):
    ctx, ctx2 = ctxs
    rng = random.Random(500 + seed)
    chk = Checker(ctx, ctx2, rng)
    wr.script(rng, chk, rounds=rng.randrange(3, 8), n_svc=rng.randrange(1, 6), churn=rng.choice([1, 3, 8]),
              flight=rng.choice([0.0, 0.1]), lib=ww_lib(ctx, rng))
    assert chk.calls >= 3 and chk.copied > 0, "nothing was ever reused"


def ww_lib(ctx, rng):
    from test_walk_watch import Lib
    return Lib(ctx, rng, full=False)


def queries(nodes):
    """a query mix over a snapshot: host A, service A, SRV with and without OPT, NODATA, NXDOMAIN"""
    out = []
    for p, data in nodes:
        name = rv.name_of(p)
        c, r = rv.classify(p, data)
        out.append(du.query(name))
        out.append(du.query(name, du.T_AAAA))
        if c == rv.OK and r[0] == "service":
            out.append(du.query(r[1] + b"." + r[2] + b"." + name, du.T_SRV))
            out.append(du.query(r[1] + b"." + r[2] + b"." + name, du.T_SRV, opt=(4096, 0, 1)))
    out.append(du.query(b"nowhere.example"))
    return out


def dns_same(ctx, ctx2, msgs):
    mb, mo = du.pack(msgs)
    for udp, tcp in ((1232, False), (512, False), (1232, True)):
        a, b = ctx.answer_dns(mb, mo, udp, tcp), ctx2.answer_dns(mb, mo, udp, tcp)
        assert a.resp.tobytes() == b.resp.tobytes() and np.array_equal(a.resp_off, b.resp_off)
        assert np.array_equal(a.status, b.status) and np.array_equal(a.tc, b.tc) and np.array_equal(a.node, b.node)
    return a


def fleet_tree(n_svc=3, n_inst=40):
    zk = ww.WalkZooKeeper()
    zk.create(b"/r", b"", 0, False)
    for s in range(n_svc):
        zk.create(b"/r/s%d" % s, service(b"_http", b"_tcp", 80, 60), 0, False)
        for i in range(n_inst):
            zk.create(b"/r/s%d/i%d" % (s, i), host(b"redis_host", b"10.1.%d.%d" % (s, i + 1), None, [6379, 6380]), 0, False)
    return zk


def test_dns_answer_parity_and_gate(ctxs):
    from registrar_b200 import _native
    ctx, ctx2 = ctxs
    zk = fleet_tree()
    ctx.walk([b"/r"], lambda fb: zk.serve(fb, SESSION), watch=True)
    ctx.walk_resolve(DH, DS)
    ctx2.resolve(ctx._walk, DH, DS)
    r = dns_same(ctx, ctx2, queries([(p, zk.nodes[p].data) for p in sorted(zk.nodes) if p.startswith(b"/r")]))
    assert r.n_status[_native.DNS_ANSWER] and r.n_status[_native.DNS_NODATA] and r.n_status[_native.DNS_NXDOMAIN]
    # a walk_refresh that rebuilt nothing keeps the answers
    ctx.walk_refresh()
    ctx.answer_dns(*du.pack([du.query(b"i1.s0.r")]))
    # a rebuilding walk_refresh, a read that appended and walk_start each close the gate
    zk.delete(b"/r/s0/i1")
    zk.create(b"/r/s0/new", host(b"redis_host", b"10.9.9.9"), 0, False)
    ctx.walk_events(np.frombuffer(zk.take_events(SESSION), np.uint8))
    ctx.walk_refresh()
    with pytest.raises(RuntimeError, match="resolve it again"):
        ctx.answer_dns(*du.pack([du.query(b"i2.s0.r")]))
    ctx.walk_resolve(DH, DS)
    ctx.answer_dns(*du.pack([du.query(b"i2.s0.r")]))
    fb, _, _ = ctx.walk_requests(100, watch=True)
    ctx.read_walk(np.frombuffer(zk.serve(fb, SESSION), np.uint8))
    with pytest.raises(RuntimeError, match="resolve it again"):
        ctx.answer_dns(*du.pack([du.query(b"i2.s0.r")]))
    ctx.walk_resolve(DH, DS)
    ctx.answer_dns(*du.pack([du.query(b"i2.s0.r")]))
    ctx.walk_start([b"/r"])
    with pytest.raises(RuntimeError, match="resolve it again"):
        ctx.answer_dns(*du.pack([du.query(b"i2.s0.r")]))
    # after a plain resolve the answers are as they always were
    ctx.resolve(_snapshot(zk), DH, DS)
    ctx.answer_dns(*du.pack([du.query(b"i2.s0.r")]))


def _snapshot(zk):
    from registrar_b200.batch import Snapshot
    return Snapshot.from_nodes([(p, zk.nodes[p].data) for p in sorted(zk.nodes) if p.startswith(b"/r")])


def test_full_cases_and_interleaved_resolve(ctxs):
    ctx, ctx2 = ctxs
    zk = fleet_tree(2, 10)
    rng = random.Random(2)
    d = wr.Driver(zk, [b"/r"], rng, ww_lib(ctx, rng))
    d.start()
    chk = Checker(ctx, ctx2, rng)
    chk(d, "first")                                             # the first call: full
    chk(d, "again")                                             # nothing changed: all copied, nothing formatted
    chk(d, "ttl", DH + 5, DS)                                   # changed default TTLs: full
    chk(d, "ttl back", DH, DS)                                  # full again (the last call's TTLs differ)
    ctx.resolve(ctx._walk, 7, 9)                                # a plain resolve in between keeps reuse
    full, fresh, copied = d.model.predict(DH, DS)
    got, counts, total = walk_resolve(ctx, DH, DS, False)
    assert counts == (0, 0, total, 0) and (full, fresh, copied) == (0, 0, total)
    d.model.resolved(DH, DS)
    d.start()                                                   # walk_start clears everything
    chk(d, "restart")


def test_reconnect_keeps_identities(ctxs):
    from test_walk_setwatches import Lib as SwLib
    ctx, ctx2 = ctxs
    rng = random.Random(3)
    zk = ws.TreeZooKeeper()
    zk.create(b"/r", b"", 0, False)
    for s in range(2):
        zk.create(b"/r/s%d" % s, service(b"_http", b"_tcp", 80, 60), 0, False)
        for i in range(6):
            zk.create(b"/r/s%d/i%d" % (s, i), host(b"redis_host", b"10.2.%d.%d" % (s, i + 1)), 0, False)
    d = wr.SwDriver(zk, [b"/r"], rng, SwLib(ctx, rng))
    d.start()
    chk = Checker(ctx, ctx2, rng)
    chk(d, "start")

    class Quiet:
        def some(self, n):
            pass
    d.drop("between", Quiet(), 0)                               # the connection drops
    zk.set_data(b"/r/s1/i2", host(b"redis_host", b"10.2.9.9"))  # changed while down
    zk.set_data(b"/r/s0/i3", zk.nodes[b"/r/s0/i3"].data)        # rewritten with the same bytes while down
    ws.check_resume(d)
    d.settle()
    assert d.model.predict(DH, DS)[:2] == (0, 1)                # only the changed node is fresh
    chk(d, "resumed")


def test_refused_call_changes_nothing(ctxs):
    import children_util as cu
    import replies_util as ru
    from registrar_b200 import _native
    ctx, ctx2 = ctxs
    zk = fleet_tree(1, 4)
    ctx.walk([b"/r"], lambda fb: zk.serve(fb, SESSION), watch=False)
    _, c0, total = walk_resolve(ctx, DH, DS, False)
    assert c0[0] == 1
    with pytest.raises(_native.RegkError, match="regk_walk_resolve: default TTLs must be >= 0"):
        ctx.walk_resolve(-1, DS)
    with pytest.raises(_native.RegkError, match="no successful regk_resolve"):
        ctx.answer_dns(*du.pack([du.query(b"i1.s0.r")]))         # a refused call leaves no answers
    _, c1, _ = walk_resolve(ctx, DH, DS, True)
    assert c1 == (0, 0, total, 0)                               # ... and keeps the text and every identity
    # a getChildren reply that lists one child twice: the next level holds that path twice
    ctx.walk_start([b"/x"])
    ctx.walk_requests(1)
    ctx.read_walk(np.frombuffer(ru.success(1, service(b"_http", b"_tcp", 80, 60)) + cu.success(2, [b"a", b"a"]), np.uint8))
    kid = host(b"redis_host", b"10.0.0.1")
    ctx.walk_requests(3)
    ctx.read_walk(np.frombuffer(ru.success(3, kid) + ru.success(4, kid) + cu.success(5, []) + cu.success(6, []), np.uint8))
    with pytest.raises(_native.RegkError) as e1:
        ctx.walk_resolve(DH, DS)
    with pytest.raises(_native.RegkError) as e2:
        ctx2.resolve(ctx._walk, DH, DS)
    assert "regk_walk_resolve: snapshot node 2 has the path of an earlier node" in str(e1.value)
    assert str(e1.value).split("snapshot node")[1] == str(e2.value).split("snapshot node")[1]
    ctx.walk_start([b"/r"])
    with pytest.raises(_native.RegkError, match="regk_walk_resolve"):
        ctx.walk_resolve(DH, -5)


def test_fleet_one_percent_churn(ctxs):
    """1 000 services x 4 000 instances; 1 % deleted, 1 % created, 1 % of addresses changed; compared with regk_resolve
    by fingerprint"""
    ctx, ctx2 = ctxs
    S, I = 1000, 4000
    zk = ww.WalkZooKeeper()
    zk.create(b"/fleet", b"", 0, False)
    for s in range(S):
        sp = b"/fleet/s%04d" % s
        zk.create(sp, service(b"_http", b"_tcp", 80, 60), 0, False)
        for i in range(I):
            zk.create(sp + b"/%07d" % i, host(b"redis_host", b"10.%d.%d.%d" % (s // 256, s % 256, i % 250), None, [6379]),
                      0, False)
    zk.take_events(7)
    ctx.walk([b"/fleet"], lambda fb: zk.serve(fb, 7), watch=True)
    first = ctx.walk_resolve(DH, DS, device=True)
    assert first.full == 1
    rng = random.Random(4)
    inst = [p for p in zk.nodes if p.count(b"/") == 3]
    n = S * I // 100
    picks = rng.sample(inst, 2 * n)
    for p in picks[:n]:
        zk.delete(p)
    for p in picks[n:]:
        zk.set_data(p, host(b"redis_host", b"10.250.%d.%d" % (rng.randrange(256), rng.randrange(250)), None, [6379]))
    for k in range(n):
        zk.create(b"/fleet/s%04d/n%07d" % (k % S, k), host(b"redis_host", b"10.200.%d.%d" % (k // 250 % 256, k % 250), None,
                                                          [6379]), 0, False)
    ctx.walk_events(np.frombuffer(zk.take_events(7), np.uint8))
    ctx.refresh_walk(lambda fb: zk.serve(fb, 7))
    out = ctx.walk_resolve(DH, DS, device=True)
    got = raw_to_dict(ctx, out.answers)
    want = _dict(ctx2.resolve(ctx._walk, DH, DS))
    fp = lambda d: {k: hashlib.sha256(np.ascontiguousarray(np.asarray(v)).tobytes()).hexdigest() for k, v in d.items()}  # noqa
    assert fp(got) == fp(want)
    assert out.full == 0 and out.n_fresh == 2 * n
    assert out.copied_bytes > 0.95 * int(out.answers.text_total)
