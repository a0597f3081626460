"""The watched heartbeat across a reconnect on the GPU: SetWatches frames of the watches the session holds
(regk_setwatches_requests) against the restatement in setwatches_util at every split, the watch kinds and the re-pend
rule, the session's zxid high-water mark, regk_read_events' SetWatches gate, and the reconnect protocol of
INTEGRATION.md §3 end to end in a ZooKeeper model whose watches die with the connection."""
import random

import numpy as np
import pytest

import children_util as cu
import events_util as eu
import reconcile_owned_util as ou
import setwatches_util as sw
from test_reconcile import _dev, run
from test_reconcile_owned import OTHER, SESSION
from test_read_replies import model_of
from test_read_events import repair

ZK_EXISTS, ZK_GETCHILDREN = 3, 8
ARM_XID, DIR_XID = 1, 2 ** 30


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


@pytest.fixture
def own(built):
    """a context of its own: the zxid high-water mark lives as long as the context, as a session's does"""
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def batch(ctx, n=3000, seed=4, records=None):
    from registrar_b200 import synth
    from registrar_b200.batch import RecordBatch
    b = RecordBatch.from_records(records) if records is not None else synth.generate("config3", n=n, seed=seed)
    return run(ctx, b)


def session_model(paths, pays, missing=()):
    zk = sw.SessionZooKeeper()
    zk.nodes = model_of(paths, pays).nodes
    for i in missing:
        zk.nodes.pop(paths[i], None)
    return zk


def dirs_of(paths):
    return [d for _, d in cu.dir_set(paths)[0]]


def arm(ctx, zk, paths):
    """round 0 with watches: every reply through read_events (the every-byte rule), then read_stats / read_children;
    -> (stats, children, bytes on the wire)"""
    fe = ctx.jute_requests(ZK_EXISTS, xid_base=ARM_XID, watch=True)[0]
    r = np.frombuffer(zk.serve_reads(fe, SESSION), np.uint8)
    assert ctx.read_events(r, xid_base=ARM_XID, n_xids=len(paths)).n_replies == len(paths)
    st = ctx.read_stats(r)
    fc = ctx.children_requests(ZK_GETCHILDREN, xid_base=DIR_XID, watch=True)[0]
    rc = np.frombuffer(zk.serve_reads(fc, SESSION), np.uint8)
    ctx.read_events(rc, xid_base=DIR_XID, n_xids=len(dirs_of(paths)))
    ch = ctx.read_children(rc)
    st.wire = fe.size + r.size + fc.size + rc.size
    return st, ch


def kinds_of(st, ch):
    return ({i: sw.stat_kind(int(e)) for i, e in enumerate(st.err)},
            {k: sw.child_kind(int(e)) for k, e in enumerate(ch.err)})


def check_frames(ctx, sg, D, E, C, rel, max_frame, lmax):
    want, off = sw.frames(D, E, C, rel, max_frame, lmax)
    assert sg.frames.tobytes() == want and sg.frame_off.tolist() == off
    limit = max_frame or sw.DEFAULT_MAX_FRAME
    assert all(b - a < limit for a, b in zip(off, off[1:]))
    assert sg.lists() == (D, E, C)


@pytest.mark.gpu
def test_frames_at_every_split(ctx):
    from registrar_b200 import _native
    paths, pays = batch(ctx)
    zk = session_model(paths, pays, missing=(5, 6, 700))
    st, ch = arm(ctx, zk, paths)
    rk, dk = kinds_of(st, ch)
    D, E, C, rr, rd = sw.lists(paths, rk, dk)
    assert D and E == [paths[5], paths[6], paths[700]] and C and not rd
    lmax = max(len(p) for p in paths)
    minimum = 32 + 2 * (4 + lmax)
    first = True
    for mf in (0, minimum, minimum + 1, 2 ** 31 - 1):
        sg = ctx.setwatches_requests(max_frame=mf)
        assert (sg.n_data, sg.n_exist, sg.n_child) == (len(D), len(E), len(C))
        assert (sg.n_repend_recs, sg.n_repend_dirs) == ((len(rr), len(rd)) if first else (0, 0))
        first = False
        check_frames(ctx, sg, D, E, C, sg.relative_zxid, mf, lmax)
        raw = ctx.setwatches_requests(max_frame=mf, device=True)
        assert _dev(ctx, raw.frames.frame_bytes, int(raw.frames.total), np.uint8).tobytes() == sg.frames.tobytes()
        assert _dev(ctx, raw.frames.frame_off, int(raw.frames.n) + 1, np.uint64).tolist() == sg.frame_off.tolist()
    assert ctx.setwatches_requests(max_frame=2 ** 31 - 1).n_frames == 1
    assert ctx.setwatches_requests(max_frame=minimum).n_frames > len(ctx.setwatches_requests().frame_off) - 1
    for mf, why in ((minimum - 1, "minimum of %d" % minimum), (2 ** 31, "2^31")):
        with pytest.raises(_native.RegkError) as e:
            ctx.setwatches_requests(max_frame=mf)
        assert e.value.code == 1 and why in e.value.message, e.value.message
    o = _native.CSetWatchesOpts(0, 1 << 5)
    import ctypes as C
    assert ctx._lib.regk_setwatches_requests(ctx._h, C.byref(o), C.byref(_native.CSetWatches())) == 1
    assert ctx._lib.regk_setwatches_requests(ctx._h, None, C.byref(_native.CSetWatches())) == 1


@pytest.mark.gpu
def test_one_entry_per_frame(ctx):
    """paths of one length, no directory armed: at the minimum every frame holds exactly one entry"""
    recs = [{"domain": b"d.example.com", "hostname": b"h%03d" % i, "type": b"host", "address": b"10.0.0.1"}
            for i in range(40)]
    paths, pays = batch(ctx, records=recs)
    zk = session_model(paths, pays)
    fe = ctx.jute_requests(ZK_EXISTS, xid_base=1, watch=True)[0]
    ctx.read_stats(np.frombuffer(zk.serve_reads(fe, SESSION), np.uint8))
    lmax = max(len(p) for p in paths)
    sg = ctx.setwatches_requests(max_frame=32 + 2 * (4 + lmax))
    assert sg.n_frames == sg.n_data == len(paths) and sg.n_repend_dirs == len(dirs_of(paths))
    check_frames(ctx, sg, list(paths), [], [], sg.relative_zxid, 32 + 2 * (4 + lmax), lmax)


@pytest.mark.gpu
def test_kinds_dups_and_errored_directories(ctx):
    recs = [{"domain": b"d%d.example.com" % (i % 2), "hostname": b"h%d" % (i % 3), "type": b"host",
             "address": b"10.0.0.%d" % i} for i in range(8)]
    paths, pays = batch(ctx, records=recs)
    zk = session_model(paths, pays, missing=(1,))
    dirs = dirs_of(paths)
    zk.nodes.pop(dirs[1], None)                                     # a directory answered NONODE
    st, ch = arm(ctx, zk, paths)
    sg = ctx.setwatches_requests()
    rk, dk = kinds_of(st, ch)
    D, E, C, rr, rd = sw.lists(paths, rk, dk)
    assert len(set(paths)) < len(paths) and len(D) + len(E) == len(set(paths))      # DUP paths listed once
    assert E == [paths[1]] and dirs[1] not in C and rd == [1]
    assert (sg.n_repend_recs, sg.n_repend_dirs, sg.n_dirty_dirs) == (0, 1, 1)
    assert sg.lists() == (D, E, C)


@pytest.mark.gpu
def test_in_flight_pending_and_a_new_batch(ctx):
    paths, pays = batch(ctx, n=2000, seed=8)
    zk = session_model(paths, pays)
    # an unread round 0 re-pends everything and frames nothing
    ctx.jute_requests(ZK_EXISTS, watch=True)
    ctx.children_requests(ZK_GETCHILDREN, watch=True)
    sg = ctx.setwatches_requests()
    nfirst = len(set(paths))
    assert sg.n_frames == 0 and sg.frames.size == 0 and sg.n_repend_recs == nfirst == sg.n_dirty_recs
    assert sg.n_repend_dirs == len(dirs_of(paths))
    # armed, then an event read and its re-check framed but not answered: that record comes back pending
    batch(ctx, n=2000, seed=8)
    st, ch = arm(ctx, zk, paths)
    zk.set_data(paths[3], b"x")
    ctx.read_events(np.frombuffer(zk.take_events(SESSION), np.uint8))
    fe = ctx.events_requests(ZK_EXISTS, xid_base=50)[0]
    assert [p for _, _, p, _ in eu.parse_reads(fe.tobytes())] == [paths[3]]
    sg = ctx.setwatches_requests()
    assert (sg.n_repend_recs, sg.n_dirty_recs, sg.n_repend_dirs) == (1, 1, 0)
    D, E, C = sg.lists()
    assert paths[3] not in D and len(D) == nfirst - 1
    assert [p for _, _, p, _ in eu.parse_reads(ctx.events_requests(ZK_EXISTS)[0].tobytes())] == [paths[3]]
    # a pending record is not listed either: it is already in the set the next re-check takes
    zk.set_data(paths[9], b"y")
    ctx.read_events(np.frombuffer(zk.take_events(SESSION), np.uint8))
    sg = ctx.setwatches_requests()
    assert paths[9] not in sg.lists()[0] and sg.n_repend_recs == 1 and sg.n_dirty_recs == 2       # 3 in flight again
    # a new batch leaves nothing listed
    batch(ctx, n=2000, seed=8)
    sg = ctx.setwatches_requests()
    assert sg.n_frames == 0 and sg.n_repend_recs == nfirst and sg.n_dirty_recs == nfirst


@pytest.mark.gpu
def test_high_water_mark_and_the_gate(own):
    from registrar_b200 import _native
    ctx = own
    paths, pays = batch(ctx, n=500, seed=3)
    base = ctx.setwatches_requests().relative_zxid
    assert base == 0

    def feed(s, xb=0, nx=0):
        return ctx.read_events(np.frombuffer(s, np.uint8), xid_base=xb, n_xids=nx)

    mark = base
    hi = max(base, 0x500000000)
    s = eu.ping() + eu.notification(paths[0], zxid=hi + 99) + cu.error(7, -101, zxid=hi) + eu.ping()
    s += cu.error(8, -101, zxid=hi + 1000)[:10]                      # a partial trailing frame
    g = feed(s, 7, 2)
    want = sw.read(s, 7, 2, mark=mark)
    assert g.partial and g.n_replies == want["n_replies"] == 1
    mark = want["mark"]
    assert mark == hi and ctx.setwatches_requests().relative_zxid == hi
    with pytest.raises(_native.RegkError):                          # a refused call leaves the mark
        feed(cu.error(7, 0, zxid=hi + 5) + cu.error(99, 0, zxid=hi + 5), 7, 1)
    assert ctx.setwatches_requests().relative_zxid == hi
    # the gate: -8 is refused as today until a SetWatches framing of this batch, then skipped and counted
    batch(ctx, n=500, seed=3)
    r8 = sw.reply(hi + 7)
    with pytest.raises(_native.RegkError) as e:
        feed(r8)
    assert "a negative xid other than -1 (notification) or -2 (ping)" in e.value.message
    ctx.setwatches_requests()
    g = feed(eu.ping() + r8 + r8)
    assert g.n_replies == 2 and g.n_pings == 1
    assert ctx.setwatches_requests().relative_zxid == hi + 7 == sw.read(r8, gate=True, mark=hi)["mark"]
    for bad, why in ((sw.reply(hi, body=b"\0\0\0\0"), "with a body"), (sw.reply(hi, err=-4), "err != 0")):
        with pytest.raises(_native.RegkError) as e:
            feed(eu.ping() + bad)
        assert "byte 20:" in e.value.message and why in e.value.message, e.value.message
        with pytest.raises(eu.Refused):
            sw.read(eu.ping() + bad, gate=True)


def stream(ctx, zk, frames, xb, n):
    r = np.frombuffer(zk.serve_reads(frames, SESSION), np.uint8)
    if n:
        ctx.read_events(r, xid_base=xb, n_xids=n)
    return r


def period(ctx, zk, xid):
    ev = ctx.read_events(np.frombuffer(zk.take_events(SESSION), np.uint8))
    fe = ctx.events_requests(ZK_EXISTS, xid_base=xid)[0]
    fc = ctx.events_requests(ZK_GETCHILDREN, xid_base=xid + 100000)[0]
    st = ctx.read_stats(stream(ctx, zk, fe, xid, len(eu.parse_reads(fe.tobytes()))))
    d = ctx.reconcile_stats(st, SESSION, zk_flags=1)
    ch = ctx.read_children(stream(ctx, zk, fc, xid + 100000, len(eu.parse_reads(fc.tobytes()))))
    return ev, st, d, ch


@pytest.mark.gpu
def test_reconnect_end_to_end(own):
    ctx = own
    paths, pays = batch(ctx, seed=21)
    gone = 50
    zk = session_model(paths, pays, missing=(gone,))
    dirs = dirs_of(paths)
    first = {}
    for i, p in enumerate(paths):
        first.setdefault(p, i)
    lone = ou.parent(paths[200])                                    # a directory deleted while the connection is down
    lone_recs = {i for p, i in first.items() if ou.parent(p) == lone}
    picks = [i for i in sorted(first.values()) if i != gone and ou.parent(paths[i]) != lone][:4]
    r_fly, r_same, r_del, r_dir = picks
    st, ch = arm(ctx, zk, paths)
    round0 = st.wire
    # 1. an event whose re-check is still in flight when the connection drops
    zk.set_data(paths[r_fly], pays[r_fly] + b" ")
    ctx.read_events(np.frombuffer(zk.take_events(SESSION), np.uint8))
    ctx.events_requests(ZK_EXISTS, xid_base=70)
    # 2. the connection drops
    zk.drop_connection(SESSION)
    sg = ctx.setwatches_requests()
    assert sg.relative_zxid == zk.zxid - 1 and sg.n_repend_recs == 1 and sg.n_repend_dirs == 0
    # 3. while it is down
    old = zk.nodes[paths[r_same]].data
    zk.set_data(paths[r_same], bytes(reversed(old)) if old != bytes(reversed(old)) else old[:-1] + b"!")
    assert len(zk.nodes[paths[r_same]].data) == len(old)
    zk.delete(paths[r_del])
    zk.create(paths[gone], pays[gone], OTHER)
    zk.create(ou.parent(paths[r_dir]) + b"/foreign", b"{}", OTHER)
    for q in [q for q in zk.nodes if ou.parent(q) == lone]:
        zk.delete(q)
    zk.delete(lone)
    # 4. reconnect: the SetWatches frames, and everything that arrives through read_events with n_xids = 0
    s = zk.serve_setwatches(sg.frames.tobytes(), SESSION)
    g = ctx.read_events(np.frombuffer(s, np.uint8))
    assert g.n_replies == sg.n_frames and not g.partial
    want_recs = {r_fly, r_same, r_del, gone} | lone_recs
    want_dirs = {dirs.index(d) for d in (ou.parent(paths[r_del]), ou.parent(paths[gone]), ou.parent(paths[r_dir]), lone)}
    fe = ctx.events_requests(ZK_EXISTS, xid_base=200)[0]
    assert [p for _, _, p, _ in eu.parse_reads(fe.tobytes())] == [paths[i] for i in sorted(want_recs)]
    fc = ctx.events_requests(ZK_GETCHILDREN, xid_base=300000)[0]
    assert [p for _, _, p, _ in eu.parse_reads(fc.tobytes())] == [dirs[k] for k in sorted(want_dirs)]
    # 5. the repair converges
    st = ctx.read_stats(stream(ctx, zk, fe, 200, len(want_recs)))
    d = ctx.reconcile_stats(st, SESSION, zk_flags=1)
    ch = ctx.read_children(stream(ctx, zk, fc, 300000, len(want_dirs)))
    # a same-length rewrite is what a stat cannot see: its re-check reads SAME
    assert d.n_create == 1 + len(lone_recs) and d.n_update == 1 and d.n_replace == 1 and ch.n_stale == 1
    ctx.mkdirp_dirs()
    fb, fo, _ = ctx.mkdirp_requests(xid_base=5000, zk_flags=0)
    assert set(zk.apply_frames(fb, fo, SESSION)) <= {ou.ZOK, ou.NODEEXISTS}
    repair(ctx, zk)
    for xid in (400, 600):
        ev, st, d, ch = period(ctx, zk, xid)
        assert d.n_create == d.n_update == d.n_replace == 0 and ch.n_stale == 0
    ev, st, d, ch = period(ctx, zk, 800)
    assert ev.n_events == 0 and st.n == 0 and ch.n_dirs == 0
    for p, i in first.items():
        assert (zk.nodes[p].data == pays[i] or i == r_same) and zk.nodes[p].owner == SESSION
    # 6. fewer bytes on the wire than re-arming by round 0
    assert sg.frames.size + len(s) < round0


@pytest.mark.gpu
def test_a_million_records_one_percent_changed(ctx):
    from registrar_b200 import synth
    b = synth.generate("config3", n=1_000_000, seed=5)
    got = ctx.register_batch(b)
    n = got.n
    paths = [got.path(i) for i in range(n)]
    first = {}
    for i, p in enumerate(paths):
        first.setdefault(p, i)
    rng = random.Random(11)
    missing = set(rng.sample(sorted(first.values()), 2000))
    # round 0 answered without a model: found or NONODE per record, every directory found
    import stats_util as su
    fe = ctx.jute_requests(ZK_EXISTS, xid_base=1, watch=True)[0]
    nodes = [eu.ru.error(su.wrap(1 + i), sw.NONODE, zxid=100) if first[paths[i]] in missing and True
             else su.success(su.wrap(1 + i), 0, 0, 2, 0, zxid=100) for i in range(n)]
    r = np.frombuffer(b"".join(nodes), np.uint8)
    assert ctx.read_events(r, xid_base=1, n_xids=n).n_replies == n
    st = ctx.read_stats(r)
    dirs = dirs_of(paths)
    fc = ctx.children_requests(ZK_GETCHILDREN, xid_base=2 ** 30, watch=True)[0]
    ctx.read_children(np.frombuffer(b"".join(cu.success(su.wrap(2 ** 30 + k), [], zxid=90) for k in range(len(dirs))),
                                    np.uint8))
    changed = rng.sample(sorted(first.values()), len(first) // 100)
    ctx.read_events(np.frombuffer(b"".join(eu.notification(paths[i], 3, zxid=200) for i in changed), np.uint8))
    sg = ctx.setwatches_requests()
    rk = {i: sw.stat_kind(int(e)) for i, e in enumerate(st.err)}
    D, E, C, rr, rd = sw.lists(paths, rk, {k: sw.CHILD for k in range(len(dirs))}, pend_recs=set(changed))
    assert not rr and not rd and sg.relative_zxid >= 100
    assert (sg.n_data, sg.n_exist, sg.n_child, sg.n_dirty_recs) == (len(D), len(E), len(C), len(changed))
    want, off = sw.frames(D, E, C, sg.relative_zxid, 0, max(len(p) for p in paths))
    assert sg.frames.tobytes() == want and sg.frame_off.tolist() == off
