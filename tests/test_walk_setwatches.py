"""A watched walk carried across a reconnect on the GPU (regk_walk_setwatches, the ARMED bit, the walk's zxid mark and
the SetWatches gate of regk_walk_events), bit for bit against walk_setwatches_util's restatement after every call,
with host and device streams and outputs alternating: frames at the default, the minimum, minimum + 1 and one entry
per frame; ARMED across plain levels, refresh levels and rebuilds, with a getChildren error and a refresh getData
error; both in-flight cases; the mark, a refused read and walk_start; the gate; the refusals, which change nothing;
random drop scripts, in lockstep and end to end through Context.resume_walk; the bytes on the wire against a full
re-walk; a million nodes at 1 % churn while the connection is down."""
import random

import numpy as np
import pytest

import events_util as ev
import setwatches_util as sw
import test_walk_watch as tw
import walk_setwatches_util as ws
import walk_watch_util as ww

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


class Lib(tw.Lib):
    """tw.Lib with walk_setwatches compared against the model: frames, offsets and every count"""

    def setwatches(self, max_frame, want):
        if self.rng.random() < 0.5:
            r = self.ctx.walk_setwatches(max_frame)
            fb, off = r.frames, r.frame_off
        else:
            r = self.ctx.walk_setwatches(max_frame, device=True)
            fr = r.frames
            fb = self.ctx._d2h(fr.frame_bytes, int(fr.total), np.uint8)
            off = self.ctx._d2h(fr.frame_off, int(fr.n) + 1, np.uint64)
        for k in ("n_listed", "n_repend", "n_pending", "n_removed", "n_frontier", "relative_zxid"):
            assert int(getattr(r, k)) == want[k], k
        if want["frames"] is None:
            listed = [p for _, D, E, C in sw.parse(fb.tobytes()) for p in D]
            assert len(listed) == want["n_listed"]
            nodes = self.full_nodes
            for k in self.rng.sample(range(len(listed)), min(2000, len(listed))):
                assert listed[k] == nodes[want["listed"][k]][0]
        else:
            assert fb.tobytes() == want["frames"] and off.tolist() == want["frame_off"]


@pytest.mark.parametrize("seed", range(16))
def test_random_drop_scripts(ctx, seed):
    rng = random.Random(2000 + seed)
    depth = [1, 2, 3, 4, 5, 6][seed % 6]
    ws.script(rng, Lib(ctx, rng), drops=rng.randrange(1, 6), depth=depth, fan=(0, 1, 2, 3) if depth > 4 else (0, 1, 2, 4),
              churn=rng.choice([2, 6, 15]), roots=[b"/z"] if seed % 3 else [b"/z", b"/y"],
              max_frame=rng.choice([0, 0, 200, 400]))


def test_frames_at_max_frame_edges(ctx):
    rng = random.Random(6)
    zk, d = ws.readme_walked(Lib(ctx, rng), rng)
    lmin = 32 + 2 * (4 + d.model.lmax())
    for mf in (0, lmin, lmin + 1, 131072, 2 ** 31 - 1):
        d.setwatches(mf)
    # one entry per frame: every path of one length, so B = 4 + P at the minimum
    zk = ws.TreeZooKeeper()
    roots = [b"/r%02d" % k for k in range(40)]
    for r in roots:
        zk.create(r, b"x", 0, False)
    d = ws.Driver(zk, roots, rng, Lib(ctx, rng))
    d.start()
    want = d.setwatches(32 + 2 * (4 + 4))
    assert len(want["frame_off"]) - 1 == 80
    for mf in (32 + 2 * 8 + 1, 0):
        d.setwatches(mf)


def test_armed_with_errors_and_rebuilds(ctx):
    """a getChildren error on a plain level and a getData error on a refresh level both leave the node unarmed, so
    setwatches re-pends it; the armed bytes move with their nodes when a refresh drops removed nodes"""
    rng = random.Random(8)
    zk = ws.TreeZooKeeper()
    ww.build_tree(zk, rng, b"/z", 3, (2, 3))
    kids = sorted(p for p in zk.nodes if p.count(b"/") == 2)
    zk.fail[(8, kids[0])] = -102
    d = ws.Driver(zk, [b"/z"], rng, Lib(ctx, rng))
    d.start()
    j0 = [n[0] for n in d.model.nodes].index(kids[0])
    assert not d.model.armed[j0]
    del zk.fail[(8, kids[0])]
    leaves = sorted(p for p in zk.nodes if not zk.kids[p] and not p.startswith(kids[0] + b"/"))
    zk.delete(leaves[0])                                       # a removed node: the rebuild renumbers the rest
    zk.set_data(kids[1], b"again")
    zk.fail[(4, kids[1])] = -102                               # its refresh getData errs: no watch
    d.feed(zk.take_events(d.SESSION))
    d.refresh()
    j1 = [n[0] for n in d.model.nodes].index(kids[1])
    assert not d.model.armed[j1] and d.model.marks[j1] == 0
    want = d.setwatches()
    assert want["n_repend"] == 2 and {j for j, mk in enumerate(d.model.marks) if mk} == {
        [n[0] for n in d.model.nodes].index(kids[0]), j1}
    del zk.fail[(4, kids[1])]
    zk.drop_connection(d.SESSION)
    d.feed(zk.serve_setwatches(want["frames"], d.SESSION))
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/z"])


@pytest.mark.parametrize("refresh", [False, True])
def test_in_flight_levels(ctx, refresh):
    """a plain level, or a refresh level, framed and answered, its replies cut off; the frontier is left alone and
    framed again after the reconnect"""
    for seed in range(6):
        rng = random.Random(300 + seed + 10 * refresh)
        zk = ws.TreeZooKeeper()
        ww.build_tree(zk, rng, b"/z", 3, (1, 2, 3))
        d = ws.Driver(zk, [b"/z"], rng, Lib(ctx, rng))
        mut = ww.Mutator(zk, [b"/z"], rng)
        d.model.start(d.roots)
        d.lib.start(d.roots)
        d.level()
        if refresh:
            d.levels()
            mut.some(3)
            d.feed(zk.take_events(d.SESSION))
            if not d.model.counts()[0]:
                continue
            d.refresh_framed()
        f = len(d.model.frontier)
        if not f:
            continue
        d.cut_level(seed % 2 == 0)
        zk.drop_connection(d.SESSION)
        mut.some(3)
        want = ws.check_resume(d)
        assert want["n_frontier"] == f
        d.levels()
        d.settle()
        assert d.snapshot_set() == zk.subtree([b"/z"])


def test_high_water_mark(ctx):
    from registrar_b200 import _native
    rng = random.Random(11)
    zk, d = ws.readme_walked(Lib(ctx, rng), rng)
    d.setwatches()                                             # relative_zxid = the largest reply zxid read
    zk.set_data(ws.PATHS_README[0], b"v2")
    # a refused read moves nothing: frame the refresh level, answer it, and offer a stream cut inside its last reply
    d.feed(zk.take_events(d.SESSION))
    d.refresh_framed()
    xb = d._next_xid(2)
    frames = d.model.requests(xb, True)
    d.lib.requests(xb, True, frames)
    zk.create(b"/us/joyent/later", b"", 0, False)              # the zxid moves on before the replies are sent
    stream = zk.serve(frames, d.SESSION)
    with pytest.raises(_native.RegkError):
        ctx.read_walk(np.frombuffer(stream[:-3], np.uint8))
    d.setwatches()                                             # the mark has not moved
    want = d.model.read(stream)
    d.lib.read(stream, want, d.model)
    d.setwatches()                                             # now it has
    assert d.model.mark == zk.zxid
    ctx.walk_start([b"/us/joyent"])                            # reset, and the gate closed
    r = ctx.walk_setwatches()
    assert (r.relative_zxid, r.n_listed, r.n_frames) == (0, 0, 0)
    ctx.walk_start([b"/us/joyent"])
    with pytest.raises(_native.RegkError, match="negative xid"):
        ctx.walk_events(np.frombuffer(sw.reply(5), np.uint8))


def test_gate(ctx):
    from registrar_b200 import _native
    rng = random.Random(12)
    zk, d = ws.readme_walked(Lib(ctx, rng), rng)
    for dev in (False, True):
        s = sw.reply(zk.zxid + 5)
        with pytest.raises(_native.RegkError, match="negative xid"):
            ctx.walk_events(tw._cuda(s) if dev else np.frombuffer(s, np.uint8))
    d.setwatches()
    for bad, what in ((sw.reply(5, body=b"x"), "with a body"), (sw.reply(5, err=-4), "err != 0")):
        with pytest.raises(_native.RegkError, match=what):
            ctx.walk_events(np.frombuffer(bad, np.uint8))
    got = d.feed(ev.notification(b"/nowhere") + sw.reply(zk.zxid + 5) + ru_ping())
    assert got["n_replies"] == 1 or got["n_pings"] == 1
    d.setwatches()                                             # the reply's zxid entered the mark
    assert d.model.mark == zk.zxid + 5


def ru_ping():
    import replies_util as ru
    return ru.ping()


def test_refusals_change_nothing(ctx):
    from registrar_b200 import _native
    c = _native.Context(0)
    try:
        with pytest.raises(_native.RegkError, match="no walk") as e:
            c.walk_setwatches()
        assert e.value.code == _native.REGK_ERR_STATE
    finally:
        c.close()
    rng = random.Random(13)
    zk = ws.TreeZooKeeper()
    ww.build_tree(zk, rng, b"/z", 2, (3,))
    d = ws.Driver(zk, [b"/z"], rng, Lib(ctx, rng))
    d.start(watch=False)
    with pytest.raises(_native.RegkError, match="unwatched") as e:
        ctx.walk_setwatches()
    assert e.value.code == _native.REGK_ERR_STATE
    zk2, d = ws.readme_walked(Lib(ctx, rng), rng)
    zk2.set_data(ws.PATHS_README[2], b"x")
    d.feed(zk2.take_events(d.SESSION))
    lmin = 32 + 2 * (4 + d.model.lmax())
    for mf in (lmin - 1, 2 ** 31, 2 ** 32 - 1):
        with pytest.raises(_native.RegkError, match="max_frame") as e:
            ctx.walk_setwatches(mf)
        assert e.value.code == _native.REGK_ERR_INVALID_ARG
    out = _native.CWalkSetWatches()
    o = _native.CSetWatchesOpts(0, 1 << 3)
    assert ctx._lib.regk_walk_setwatches(ctx._h, _native.C.byref(o), _native.C.byref(out)) == _native.REGK_ERR_INVALID_ARG
    with pytest.raises(_native.RegkError, match="negative xid"):  # no gate yet
        ctx.walk_events(np.frombuffer(sw.reply(1), np.uint8))
    want = d.setwatches()                                      # and nothing changed: the model agrees
    assert want["n_pending"] == 1


def _fresh_walk_bytes(zk, roots):
    from registrar_b200 import _native
    c, n = _native.Context(0), [0]
    try:
        def exchange(fb):
            s = zk.serve(fb, 7)
            n[0] += len(fb) + len(s)
            return s
        c.walk(roots, exchange, watch=True)
    finally:
        c.close()
    return n[0]


@pytest.mark.parametrize("seed", range(6))
def test_resume_walk_end_to_end(ctx, seed):
    """Context.walk, the connection dropped (sometimes mid-level), the tree changed, Context.resume_walk and
    refresh_walk to convergence; fewer bytes on the wire than a full re-walk of the same state"""
    rng = random.Random(500 + seed)
    zk = ws.TreeZooKeeper()
    ww.build_tree(zk, rng, b"/z", 4, (1, 2, 4))
    mut = ww.Mutator(zk, [b"/z"], rng)
    session, wire = 41, [0]

    def exchange(fb):
        fb = bytes(fb)
        s = zk.serve_setwatches(fb, session) if ev_is_setwatches(fb) else zk.serve(fb, session)
        wire[0] += len(fb) + len(s)
        return s
    if seed % 2:
        ctx.walk([b"/z"], exchange, watch=True)
    else:                                                      # drop with the second level in flight
        ctx.walk_start([b"/z"])
        fb = ctx.walk_requests(1, watch=True)[0]
        s = zk.serve(fb.tobytes(), session)
        ctx.read_walk(np.frombuffer(s, np.uint8))
        ctx.walk_events(np.frombuffer(s, np.uint8), 0, 1, 2)
        fb = ctx.walk_requests(3, watch=True)[0]
        zk.serve(fb.tobytes(), session)                        # answered, never delivered
    zk.drop_connection(session)
    mut.some(4)
    wire[0] = 0
    r, w = ctx.resume_walk(exchange, xid_base=100)
    for _ in range(50):
        e = ctx.walk_events(np.frombuffer(zk.take_events(session), np.uint8))
        if e.n_pending == 0 and e.n_removed == 0:
            break
        _, w = ctx.refresh_walk(exchange, xid_base=1000)
    s = w.snapshot()
    pb, jb, po, jo = s.path_bytes.tobytes(), s.json_bytes.tobytes(), s.path_off.tolist(), s.json_off.tolist()
    got = {(pb[po[j]:po[j + 1]], jb[jo[j]:jo[j + 1]], int(s.version[j]), int(s.owner[j])) for j in range(w.m)}
    assert got == zk.subtree([b"/z"]) and len(got) == w.m
    if seed % 2:
        assert wire[0] < _fresh_walk_bytes(zk, [b"/z"])
    with pytest.raises(ValueError, match="SetWatches replies"):
        ctx.resume_walk(lambda fb: b"")


def ev_is_setwatches(fb):
    return len(fb) >= 12 and fb[4:12] == b"\xff\xff\xff\xf8\x00\x00\x00\x65"


@pytest.mark.slow
def test_million_nodes_one_percent_churn_while_down(ctx):
    """1 000 service records x 1 000 instances walked with watches; the connection drops; 1 % of the instances
    deleted, as many created and every tenth service record rewritten while it is down; SetWatches, its events,
    one refresh: counts exact and a sampled comparison"""
    from test_resolve_cpu import host, service
    rng = random.Random(21)
    zk = ws.TreeZooKeeper()
    zk.create(b"/fleet", b"", 0, False)
    for s in range(1000):
        sp = b"/fleet/s%03d" % s
        zk.create(sp, service(b"_http", b"_tcp", 80, 60), 0, False)
        for i in range(1000):
            zk.create(sp + b"/%06d" % i, host(b"redis_host", b"10.%d.%d.%d" % (s // 256, s % 256, i % 250), None, [6379]),
                      0, False)
    lib = Lib(ctx, rng, full=False)
    d = ws.Driver(zk, [b"/fleet"], rng, lib)
    d.start()
    assert len(d.model.nodes) == 1_001_001
    zk.drop_connection(d.SESSION)
    inst = [p for p in zk.nodes if p.count(b"/") == 3]
    for p in rng.sample(inst, 5000):
        zk.delete(p)
    for k in range(5000):
        zk.create(b"/fleet/s%03d/n%05d" % (k % 1000, k), host(b"redis_host", b"10.200.0.%d" % (k % 250), None, [6379]), 0,
                  False)
    for s in range(0, 1000, 10):
        zk.set_data(b"/fleet/s%03d" % s, service(b"_http", b"_tcp", 8080, 60))
    lib.full_nodes = d.model.nodes
    want = d.model.setwatches(0, frames=False)
    lib.setwatches(0, want)
    assert want["n_listed"] == 1_001_001
    r = ctx.walk_setwatches()                                  # the framing again, for the stream the server answers
    stream = zk.serve_setwatches(r.frames.tobytes(), d.SESSION)
    d.feed(stream)
    assert d.model.counts() == (1000, 5000)                     # every service's pzxid moved
    out = d.refresh()
    assert (out["n_removed"], out["n_frontier"]) == (5000, 1000)
    d.settle()
    w, nodes = d.lib.w, d.model.nodes
    s = w.snapshot()
    po, jo = s.path_off, s.json_off
    for j in rng.sample(range(w.m), 2000) + [0, w.m - 1]:
        assert s.path_bytes[po[j]:po[j + 1]].tobytes() == nodes[j][0]
        assert s.json_bytes[jo[j]:jo[j + 1]].tobytes() == nodes[j][1]
    assert set(nodes) == zk.subtree([b"/fleet"])
