"""The watched walk on the GPU (regk_walk_requests with REGK_ZK_WATCH, regk_walk_events, regk_walk_refresh and the
refresh level of regk_read_walk), bit for bit against walk_watch_util's restatement after every call: frames, event
arrays and counts, snapshot streams, versions, owners, level_off, frontier and every counter.  The README tree; random
trees over many churn rounds with mutations landing inside reply streams; host and device streams and outputs; streams
fed in two pieces; refusals that change nothing; the state rules; resolve on a refreshed snapshot against resolve on a
fresh walk; a million nodes under a thousand service records at 1 % churn."""
import random

import numpy as np
import pytest

import events_util as ev
import walk_util as wu
import walk_watch_util as ww
from test_resolve_cpu import host, service

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def _cuda(b):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(b), np.uint8).copy()).cuda()


class Lib:
    """the library in lockstep with the model, compared after every call; device streams and outputs alternate"""

    def __init__(self, ctx, rng, full=True):
        self.ctx, self.rng, self.full, self.w = ctx, rng, full, None

    def start(self, roots):
        self.ctx.walk_start(roots)

    def requests(self, xid, watch, frames):
        if self.rng.random() < 0.5:
            got = self.ctx.walk_requests(xid, watch=watch)[0]
        else:
            out = self.ctx.walk_requests(xid, device=True, watch=watch)
            got = self.ctx._d2h(out.frame_bytes, int(out.total), np.uint8)
        assert got.tobytes() == frames

    def read(self, stream, want, model):
        self.w = self.ctx.read_walk(_cuda(stream) if self.rng.random() < 0.5 else np.frombuffer(stream, np.uint8))
        for k, v in want.items():
            assert getattr(self.w, k) == v, k
        self.check(model, self.w)

    def events(self, stream, start, xid_base, n_xids, want):
        dev_in, dev_out = self.rng.random() < 0.5, self.rng.random() < 0.3
        s = _cuda(stream) if dev_in and stream else np.frombuffer(stream, np.uint8)
        raw = self.ctx.walk_events(s, start, xid_base, n_xids, device=dev_out)
        got = raw_events(self.ctx, raw) if dev_out else raw
        for k in ("n_events", "n_pings", "n_replies", "n_unmatched", "n_other", "consumed", "partial", "n_pending",
                  "n_removed"):
            assert getattr(got, k) == want[k], k
        assert list(zip(got.pos.tolist(), got.type.tolist(), got.state.tolist(), got.zxid.tolist(),
                        got.node.tolist())) == want["events"]

    def refresh(self, want, model):
        r = self.ctx.walk_refresh()
        assert (r.n_removed, r.n_kept, r.n_frontier) == (want["n_removed"], want["n_kept"], want["n_frontier"])
        self.w = r.walk
        self.check(model, r.walk)

    def check(self, model, w):
        assert w.m == len(model.nodes) and w.level_off.tolist() == model.level_off
        assert w.n_frontier == len(model.frontier)
        if not self.full and w.m > 5000:
            return
        s = w.snapshot()
        pb, jb, po, jo = s.path_bytes.tobytes(), s.json_bytes.tobytes(), s.path_off.tolist(), s.json_off.tolist()
        assert [pb[po[j]:po[j + 1]] for j in range(w.m)] == [n[0] for n in model.nodes]
        assert [jb[jo[j]:jo[j + 1]] for j in range(w.m)] == [n[1] for n in model.nodes]
        assert s.version.tolist() == [n[2] for n in model.nodes] and s.owner.tolist() == [n[3] for n in model.nodes]


class _Raw:
    pass


def raw_events(ctx, raw):
    """a device CWalkEvents copied to the host, shaped as WalkEvents"""
    g, n = _Raw(), int(raw.n_events)
    for k in ("n_events", "n_pings", "n_replies", "n_unmatched", "n_other", "consumed", "n_pending", "n_removed"):
        setattr(g, k, int(getattr(raw, k)))
    g.partial = bool(raw.partial)
    g.pos, g.type = ctx._d2h(raw.pos, n, np.uint64), ctx._d2h(raw.type, n, np.int32)
    g.state, g.zxid = ctx._d2h(raw.state, n, np.int32), ctx._d2h(raw.zxid, n, np.int64)
    g.node = ctx._d2h(raw.node, n, np.uint64)
    return g


@pytest.mark.parametrize("seed", range(12))
def test_random_scripts(ctx, seed):
    rng = random.Random(1000 + seed)
    depth = [1, 2, 3, 4, 5, 6, 8][seed % 7]
    ww.script(rng, Lib(ctx, rng), rounds=rng.randrange(4, 12), depth=depth,
              fan=(0, 1, 2, 3) if depth > 4 else (0, 1, 2, 4, 9), churn=rng.choice([2, 6, 20]),
              flight=rng.choice([0.0, 0.05, 0.3]), roots=[b"/z"] if seed % 3 else [b"/z", b"/y"])


def test_delete_recreate_race(ctx):
    """walk_watch_util.spent_watch_race through the library: p's NodeDeleted makes g pending, and the next refresh
    walks the new p"""
    rng = random.Random(4)
    d = ww.spent_watch_race(Lib(ctx, rng))
    assert d.model.counts() == (1, 1)
    d.settle()
    assert (b"/z/g/p", b"p2", 0, 0) in d.snapshot_set() and d.snapshot_set() == d.zk.subtree([b"/z"])


def test_readme_tree(ctx):
    """the authcache tree walked with watches; an instance deleted, one added and the service record rewritten;
    refreshed; resolve on it equals resolve on a fresh walk"""
    rng = random.Random(3)
    zk = ww.WalkZooKeeper()
    t = wu.readme_tree()
    for p in sorted(t.nodes, key=len):
        zk.create(p, t.nodes[p][0], 0, False)
    d = ww.Driver(zk, [b"/us/joyent"], rng, Lib(ctx, rng))
    d.start()
    inst = sorted(p for p in zk.nodes if p.count(b"/") == 5)
    zk.delete(inst[0])
    zk.create(b"/us/joyent/emy-10/authcache/new", host(b"redis_host", b"10.99.99.31", None, [6379]), 0, False)
    zk.set_data(b"/us/joyent/emy-10/authcache", service(b"_redis", b"_tcp", 6380, 60))
    d.feed(zk.take_events(d.SESSION))
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/us/joyent"])
    same_answers(ctx, d)


def answer_sets(a):
    out = {}
    for q in range(a.n_queries):
        lines = a.answer(q) + a.additional(q)
        out.setdefault(int(a.q_kind[q]), []).append(frozenset(lines.split(b"\n")))
    return {k: sorted(v, key=sorted) for k, v in out.items()}


def same_answers(ctx, d):
    """resolve on the refreshed snapshot against resolve on a fresh walk of the same tree, as sets of answer lines"""
    from registrar_b200 import _native
    a1 = ctx.resolve(d.lib.w, 30, 60)
    c2 = _native.Context(0)
    try:
        w2 = c2.walk(d.roots, lambda fb: d.zk.serve(fb, 1))
        a2 = c2.resolve(w2, 30, 60)
        assert answer_sets(a1) == answer_sets(a2)
    finally:
        c2.close()


def test_resolve_after_churn(ctx):
    rng = random.Random(77)
    zk = ww.WalkZooKeeper()
    zk.create(b"/us", b"", 0, False)
    zk.create(b"/us/zone", b"", 0, False)
    for s in range(20):
        sp = b"/us/zone/svc%d" % s
        zk.create(sp, service(b"_http", b"_tcp", 8000 + s, 60), 0, False)
        for i in range(rng.randrange(0, 12)):
            zk.create(sp + b"/i%d" % i, host(b"redis_host", b"10.0.%d.%d" % (s, i), None, [8000 + s]), 0, False)
    d = ww.Driver(zk, [b"/us"], rng, Lib(ctx, rng))
    d.start()
    for r in range(5):
        svcs = [b"/us/zone/svc%d" % s for s in range(20)]
        for _ in range(6):
            sp = rng.choice(svcs)
            kids = list(zk.kids[sp])
            if kids and rng.random() < 0.5:
                zk.delete(sp + b"/" + rng.choice(kids))
            else:
                zk.create(sp + b"/r%d_%d" % (r, rng.randrange(10 ** 6)),
                          host(b"redis_host", b"10.1.%d.%d" % (r, rng.randrange(256)), None, [80]), 0, False)
        zk.set_data(rng.choice(svcs), service(b"_http", b"_tcp", 9000 + r, 30))
        d.feed(zk.take_events(d.SESSION))
        d.refresh()
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/us"])
    same_answers(ctx, d)


def test_refusals_change_nothing(ctx):
    from registrar_b200 import _native
    rng = random.Random(5)
    zk = ww.WalkZooKeeper()
    ww.build_tree(zk, rng, b"/z", 3, (2, 3))
    lib = Lib(ctx, rng)
    d = ww.Driver(zk, [b"/z"], rng, lib)
    d.start()
    leaves = [p for p in zk.nodes if not zk.kids[p]]
    zk.delete(leaves[0])
    zk.set_data(leaves[1], b"x")
    good = zk.take_events(d.SESSION)
    bads = [good + ev.notification(b"/z", 9),                  # a type outside -1 .. 7
            good + ev.notification(b"/z", plen=-1),
            ev.notification(b"/z", err=-4) + good,
            good + ru_error(77)]                               # a reply outside the range
    for bad in bads:
        for dev in (False, True):
            with pytest.raises(_native.RegkError, match="regk_walk_events: byte [0-9]+"):
                ctx.walk_events(_cuda(bad) if dev else np.frombuffer(bad, np.uint8))
            with pytest.raises(ev.Refused):
                ww.Model.events(d.model, bad)
    d.feed(good)                                               # nothing was marked: the corrected stream reads as new
    assert d.model.counts() == (2, 1)
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/z"])


def ru_error(xid):
    import replies_util as ru
    return ru.error(xid, 0)


def test_state_rules(ctx):
    from registrar_b200 import _native
    rng = random.Random(9)
    zk = ww.WalkZooKeeper()
    ww.build_tree(zk, rng, b"/z", 2, (3,))
    with_lib = ww.Driver(zk, [b"/z"], rng, Lib(ctx, rng))
    with_lib.start(watch=False)                                # an unwatched walk
    for call in (lambda: ctx.walk_events(np.zeros(0, np.uint8)), ctx.walk_refresh):
        with pytest.raises(_native.RegkError, match="unwatched") as e:
            call()
        assert e.value.code == _native.REGK_ERR_STATE
    ctx.walk_start([b"/z"])                                    # a level outstanding
    fb = ctx.walk_requests(1, watch=True)[0]
    with pytest.raises(_native.RegkError, match="outstanding") as e:
        ctx.walk_refresh()
    assert e.value.code == _native.REGK_ERR_STATE
    ctx.read_walk(np.frombuffer(zk.serve(fb, 2), np.uint8))
    fb = ctx.walk_requests(7, watch=False)[0]                  # the last framing counts: this level is unwatched
    ctx.read_walk(np.frombuffer(zk.serve(fb, 2), np.uint8))
    with pytest.raises(_native.RegkError, match="unwatched"):
        ctx.walk_refresh()
    d = ww.Driver(zk, [b"/z"], rng, Lib(ctx, rng))             # walk_start drops every mark and the refresh state
    d.start()
    zk.set_data(b"/z", b"changed")
    d.feed(zk.take_events(ww.Driver.SESSION))
    assert d.model.counts() == (1, 0)
    ctx.walk_start([b"/z"])
    d2 = ww.Driver(zk, [b"/z"], rng, Lib(ctx, rng))
    d2.start()
    assert ctx.walk_refresh().n_frontier == 0
    with pytest.raises(_native.RegkError, match="flags"):
        ctx._check(ctx._lib.regk_walk_refresh(ctx._h, 1, _native.C.byref(_native.CWalkRefresh())))


def test_python_loop(ctx):
    """Context.walk(watch=True) and refresh_walk() over an exchange that mutates the tree between rounds"""
    rng = random.Random(31)
    zk = ww.WalkZooKeeper()
    ww.build_tree(zk, rng, b"/z", 4, (0, 1, 3))
    mut = ww.Mutator(zk, [b"/z"], rng)
    session = 99

    def exchange(fb):
        return zk.serve(fb, session, mut.in_flight(0.1))
    ctx.walk([b"/z"], exchange, watch=True)
    for _ in range(8):
        mut.some(5)
        ctx.walk_events(np.frombuffer(zk.take_events(session), np.uint8))
        ctx.refresh_walk(exchange)
    ctx.walk_events(np.frombuffer(zk.take_events(session), np.uint8))
    for _ in range(50):
        r, w = ctx.refresh_walk(exchange)
        e = ctx.walk_events(np.frombuffer(zk.take_events(session), np.uint8))
        if r.n_frontier == 0 and r.n_removed == 0 and e.n_pending == 0 and e.n_removed == 0:
            break
    s = w.snapshot()
    pb, jb, po, jo = s.path_bytes.tobytes(), s.json_bytes.tobytes(), s.path_off.tolist(), s.json_off.tolist()
    got = {(pb[po[j]:po[j + 1]], jb[jo[j]:jo[j + 1]], int(s.version[j]), int(s.owner[j])) for j in range(w.m)}
    assert got == zk.subtree([b"/z"]) and len(got) == w.m


@pytest.mark.slow
def test_million_nodes_one_percent_churn(ctx):
    """1 000 service records x 1 000 instances walked with watches; half of 1 % of the instances deleted, as many
    created, and every service record rewritten; refreshed; counts exact and a sampled comparison"""
    rng = random.Random(12)
    zk = ww.WalkZooKeeper()
    zk.create(b"/fleet", b"", 0, False)
    for s in range(1000):
        sp = b"/fleet/s%03d" % s
        zk.create(sp, service(b"_http", b"_tcp", 80, 60), 0, False)
        for i in range(1000):
            zk.create(sp + b"/%06d" % i, host(b"redis_host", b"10.%d.%d.%d" % (s // 256, s % 256, i % 250), None, [6379]),
                      0, False)
    zk.take_events(ww.Driver.SESSION)
    d = ww.Driver(zk, [b"/fleet"], rng, Lib(ctx, rng, full=False))
    d.start()
    assert len(d.model.nodes) == 1_001_001
    inst = [p for p in zk.nodes if p.count(b"/") == 3]
    for p in rng.sample(inst, 5000):
        zk.delete(p)
    for k in range(5000):
        zk.create(b"/fleet/s%03d/n%05d" % (k % 1000, k), host(b"redis_host", b"10.200.0.%d" % (k % 250), None, [6379]), 0,
                  False)
    for s in range(1000):
        zk.set_data(b"/fleet/s%03d" % s, service(b"_http", b"_tcp", 8080, 60))
    d.feed(zk.take_events(d.SESSION))
    assert d.model.counts() == (1000, 5000)
    r = d.refresh()
    assert (r["n_removed"], r["n_frontier"]) == (5000, 1000)
    assert d.model.counts() == (0, 0)
    w = d.lib.w
    nodes = d.model.nodes
    s = w.snapshot()
    po, jo = s.path_off, s.json_off
    for j in rng.sample(range(w.m), 2000) + [0, w.m - 1]:
        assert s.path_bytes[po[j]:po[j + 1]].tobytes() == nodes[j][0]
        assert s.json_bytes[jo[j]:jo[j + 1]].tobytes() == nodes[j][1]
        assert (int(s.version[j]), int(s.owner[j])) == (nodes[j][2], nodes[j][3])
    assert set(nodes) == zk.subtree([b"/fleet"])
