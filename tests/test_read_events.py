"""The watched heartbeat on the GPU: watch-byte framings (REGK_ZK_WATCH), the session stream read into events mapped to
records and service directories (regk_read_events), the re-arming re-checks of only what fired (regk_events_requests)
read as subsets by regk_read_stats / regk_reconcile_stats / regk_read_children, every output against the restatement
in events_util, and the watched loop of INTEGRATION.md §3 end to end in the watch-aware ZooKeeper model."""
import ctypes as C
import random

import numpy as np
import pytest

import children_util as cu
import events_util as eu
import reconcile_owned_util as ou
import stats_util as su
from test_reconcile import _dev, run
from test_reconcile_owned import OTHER, SESSION
from test_read_replies import model_of

ZK_CREATE, ZK_DELETE, ZK_EXISTS, ZK_GETDATA, ZK_SETDATA, ZK_GETCHILDREN, ZK_REPLACE = 1, 2, 3, 4, 5, 8, 256


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def dirs_of(paths):
    return [d for _, d in cu.dir_set(paths)[0]]


def watched_model(paths, pays):
    zk = eu.WatchedZooKeeper()
    base = model_of(paths, pays)
    zk.nodes = base.nodes
    return zk


def check(ctx, paths, stream, start=0, xb=0, nx=0):
    """read_events over a host and a device copy of `stream` (fresh pending sets each: a new batch generation drops
    them) against the restatement; returns the host Events"""
    import torch
    want = eu.read(stream, xb, nx, start)
    m = eu.Mapper(paths)
    subj, unmatched, other = m.feed(want["events"])
    a = np.frombuffer(stream, np.uint8)
    got = None
    for dev in (False, True):
        ctx.register_batch(ctx._last_batch)
        g = ctx.read_events(torch.from_numpy(a.copy()).cuda() if dev else a, start=start, xid_base=xb, n_xids=nx)
        assert g.pos.tolist() == [e[0] for e in want["events"]]
        assert g.type.tolist() == [e[1] for e in want["events"]] and g.state.tolist() == [e[2] for e in want["events"]]
        assert g.zxid.tolist() == [e[3] for e in want["events"]]
        assert list(zip(g.subject_kind.tolist(), g.subject.tolist())) == subj
        assert (g.n_events, g.n_pings, g.n_replies, g.n_unmatched, g.n_other) == (
            len(want["events"]), want["n_pings"], want["n_replies"], unmatched, other)
        assert (g.consumed, g.partial) == (want["consumed"], want["partial"])
        assert (g.n_dirty_recs, g.n_dirty_dirs) == (len(m.dirty_recs), len(m.dirty_dirs))
        got = got or g
    raw = ctx.read_events(a, start=start, xid_base=xb, n_xids=nx, device=True)
    assert np.array_equal(_dev(ctx, raw.subject, got.n_events, np.uint64), got.subject)
    return got, m


def batch(ctx, n=3000, seed=4):
    from registrar_b200 import synth
    b = synth.generate("config3", n=n, seed=seed)
    ctx._last_batch = b
    return run(ctx, b)


@pytest.mark.gpu
def test_watch_byte_frames(ctx):
    from registrar_b200 import _native
    paths, pays = batch(ctx)
    for op in (ZK_EXISTS, ZK_GETDATA):
        for w in (False, True):
            assert ctx.jute_requests(op, xid_base=9, watch=w)[0].tobytes() == eu.read_frames(op, paths, 9, watch=w)
    for w in (False, True):
        assert ctx.children_requests(ZK_GETCHILDREN, xid_base=-5, watch=w)[0].tobytes() == \
            eu.read_frames(8, dirs_of(paths), -5, watch=w)
    for op in (ZK_CREATE, ZK_DELETE, ZK_SETDATA):
        with pytest.raises(_native.RegkError) as e:
            ctx.jute_requests(op, watch=True)
        assert e.value.code == 1 and "REGK_ZK_WATCH" in e.value.message
    ctx.reconcile_stats(ctx.read_stats(np.frombuffer(su.replies(model_of(paths, pays),
                                                                ctx.jute_requests(ZK_EXISTS)[0]), np.uint8)), SESSION)
    o = _native.CJuteOpts(ZK_SETDATA, _native.FLAG_ZK_WATCH, 1, 0, -1, 0)
    assert ctx._lib.regk_reconcile_requests(ctx._h, C.byref(o), C.byref(_native.CFrames())) == 1
    ctx.read_children(np.frombuffer(cu.replies(model_of(paths, pays), ctx.children_requests()[0]), np.uint8))
    with pytest.raises(_native.RegkError) as e:
        ctx.children_requests(ZK_DELETE, watch=True)
    assert e.value.code == 1


def stream_of(paths, rng, xb=100, nx=50, count=400):
    """notifications of every type for records (DUP paths included), directories, the directories' ancestors and
    unknown paths, with pings and in-range replies between them"""
    dirs = dirs_of(paths)
    parts = []
    for _ in range(count):
        c = rng.randrange(10)
        if c == 0:
            parts.append(eu.ping())
        elif c == 1:
            parts.append(su.error(su.wrap(xb + rng.randrange(nx)), su.NONODE) if rng.randrange(2) else
                         su.success(su.wrap(xb + rng.randrange(nx)), 1, 2, 3, seed=c))
        elif c < 6:
            parts.append(eu.notification(rng.choice(paths), rng.choice([1, 2, 3, 3, 4]), zxid=rng.getrandbits(40)))
        elif c < 8:
            parts.append(eu.notification(rng.choice(dirs), rng.choice([2, 4, 4, 3]), state=rng.choice([3, 0])))
        elif c == 8:
            parts.append(eu.notification(rng.choice([b"", b"/", b"/nothere", rng.choice(paths) + b"x"]), rng.choice([-1, 0, 1, 5, 6, 7])))
        else:
            parts.append(eu.notification(rng.choice(paths)[:-1], 3))
    return b"".join(parts)


@pytest.mark.gpu
def test_streams_at_every_start_phase_with_pings_and_replies(ctx):
    from registrar_b200.batch import RecordBatch
    paths, pays = batch(ctx)
    s = stream_of(paths, random.Random(1))
    for phase in range(16):
        front = eu.ping() * 2 + bytes(range(phase))
        g, _ = check(ctx, paths, front + s, start=len(front), xb=100, nx=50)
        assert g.n_events and g.n_pings and g.n_replies and g.n_unmatched and g.n_other and g.n_dirty_dirs
    # a partial trailing frame, and xids that wrap
    for cut in (1, 3, 4, 20, 31):
        g, _ = check(ctx, paths, s + eu.notification(b"/q/r", 3)[:cut], xb=100, nx=50)
        assert g.partial and g.consumed == len(s)
    check(ctx, paths, su.error(-2 ** 31, 0) + eu.notification(paths[0]) + su.error(2 ** 31 - 1, 1), xb=2 ** 31 - 1, nx=2)
    check(ctx, paths, b"")
    # DUP paths: the first record is the subject
    recs = [{"domain": b"d.example.com", "hostname": b"h%d" % (i % 3), "type": b"host", "address": b"10.0.0.%d" % i}
            for i in range(6)]
    b = RecordBatch.from_records(recs)
    ctx._last_batch = b
    paths, _ = run(ctx, b)
    g, _ = check(ctx, paths, b"".join(eu.notification(p, 3) for p in paths))
    assert g.subject.tolist() == [0, 1, 2, 0, 1, 2] and g.n_dirty_recs == 3


@pytest.mark.gpu
def test_chunks_accumulate_and_a_new_batch_drops_them(ctx):
    paths, pays = batch(ctx)
    s = stream_of(paths, random.Random(2), count=600)
    rng = random.Random(3)
    want = eu.Mapper(paths)
    want.feed(eu.read(s, 100, 50)["events"])
    a = np.frombuffer(s, np.uint8)
    pos = 0
    while pos < len(s):
        end = min(len(s), pos + rng.randrange(1, 700))
        g = ctx.read_events(a[:end], start=pos, xid_base=100, n_xids=50)
        pos = g.consumed
    counts = (len(want.dirty_recs), len(want.dirty_dirs))
    assert (g.n_dirty_recs, g.n_dirty_dirs) == counts
    fe = ctx.events_requests(ZK_EXISTS, xid_base=7)[0].tobytes()
    assert fe == eu.read_frames(3, [paths[i] for i in want.take()], 7, watch=True)
    fc = ctx.events_requests(ZK_GETCHILDREN, xid_base=70)[0].tobytes()
    dirs = dirs_of(paths)
    assert fc == eu.read_frames(8, [dirs[k] for k in want.take(dirs=True)], 70, watch=True)
    assert ctx.events_requests(ZK_EXISTS)[0].size == 0                              # taken
    g = ctx.read_events(a, xid_base=100, n_xids=50)                                 # the next epoch marks them afresh
    assert (g.n_dirty_recs, g.n_dirty_dirs) == counts
    ctx.register_batch(ctx._last_batch)                                             # a new batch drops the pending set
    from registrar_b200 import _native
    with pytest.raises(_native.RegkError) as e:
        ctx.events_requests(ZK_EXISTS)
    assert e.value.code == 5
    assert ctx.read_events(np.zeros(0, np.uint8)).n_dirty_recs == 0
    assert ctx.events_requests(ZK_EXISTS)[0].size == 0


@pytest.mark.gpu
def test_refusals(ctx):
    from registrar_b200 import _native
    paths, _ = batch(ctx, n=500)
    good = eu.notification(paths[0]) + eu.ping()
    cases = [(eu.notification(b"/a", err=-4), "err != 0"), (eu.notification(b"/a", typ=8), "type"),
             (eu.notification(b"/abc", plen=-1), "negative path length"), (eu.notification(b"/abc", plen=2), "28 +"),
             (su.error(-2, 0) + b"\0" * 4, None), (su.error(-3, 0), "negative xid"), (su.error(5, 0), "reply range"),
             (b"\0\0\0\x0f" + b"\0" * 15, "below 16")]
    bad = bytearray(su.error(-2, 0))
    bad[0:4] = b"\0\0\0\x14"
    cases[4] = (bytes(bad) + b"\0" * 4, "ping with a body")
    for frame, why in cases:
        s = good + frame
        with pytest.raises(_native.RegkError) as e:
            ctx.read_events(np.frombuffer(s, np.uint8), xid_base=100, n_xids=3)
        assert e.value.code == 1 and ("byte %d:" % len(good)) in e.value.message and why in e.value.message, e.value.message
        with pytest.raises(eu.Refused):
            eu.read(s, 100, 3)
    assert ctx.read_events(np.frombuffer(good, np.uint8)).n_dirty_recs == 1      # a refused stream marked nothing
    for xb, nx in ((-5, 5), (-1, 1), (2 ** 31 - 1, 2 ** 32 - 1)):
        with pytest.raises(_native.RegkError) as e:
            ctx.read_events(np.frombuffer(good, np.uint8), xid_base=xb, n_xids=nx)
        assert e.value.code == 1
    with pytest.raises(_native.RegkError) as e:
        ctx.read_events(np.frombuffer(good, np.uint8), start=len(good) + 1)
    assert e.value.code == 1
    for op in (ZK_CREATE, ZK_GETDATA, ZK_DELETE):
        with pytest.raises(_native.RegkError) as e:
            ctx.events_requests(op)
        assert e.value.code == 1


def serve(zk, frames):
    return np.frombuffer(zk.serve_reads(frames, SESSION), np.uint8)


def drift(zk, paths, pays):
    """a foreign delete, a setData of another length, an ephemeral owned by another session, a new stale child"""
    zk.delete(paths[10])
    zk.set_data(paths[12], pays[12] + b"  ")
    zk.delete(paths[14])
    zk.create(paths[14], pays[14], OTHER)
    zk.create(ou.parent(paths[20]) + b"/stale-instance", b"{}", OTHER)


def arm(ctx, zk):
    ctx.read_stats(serve(zk, ctx.jute_requests(ZK_EXISTS, xid_base=1, watch=True)[0]))
    ctx.read_children(serve(zk, ctx.children_requests(ZK_GETCHILDREN, xid_base=2 ** 30, watch=True)[0]))


@pytest.mark.gpu
def test_subset_reads_equal_the_full_round(ctx):
    from registrar_b200 import _native
    paths, pays = batch(ctx)
    zk = watched_model(paths, pays)
    arm(ctx, zk)
    drift(zk, paths, pays)
    s = zk.take_events(SESSION)
    g = ctx.read_events(np.frombuffer(s, np.uint8))
    m = eu.Mapper(paths)
    m.feed(eu.read(s)["events"])
    assert (g.n_dirty_recs, g.n_dirty_dirs) == (len(m.dirty_recs), len(m.dirty_dirs)) and g.n_dirty_dirs
    fe = ctx.events_requests(ZK_EXISTS, xid_base=500)[0]
    dirty = m.take()
    assert [p for _, _, p, w in eu.parse_reads(fe.tobytes())] == [paths[i] for i in dirty]
    st = ctx.read_stats(serve(zk, fe))
    assert st.n == len(dirty)
    with pytest.raises(_native.RegkError) as e:
        ctx.reconcile_stats(st, SESSION, known_mzxid=np.zeros(st.n, np.int64))
    assert e.value.code == 1
    d_sub = ctx.reconcile_stats(st, SESSION)
    fc = ctx.events_requests(ZK_GETCHILDREN, xid_base=900)[0]
    sub_dirs = [p for _, _, p, w in eu.parse_reads(fc.tobytes()) if w == 1]
    ch_sub = ctx.read_children(serve(zk, fc))
    lst_sub, stale_sub = ch_sub.listing(), ch_sub.stale_paths()                    # valid until the next read_children
    # the full rounds over the same model state, without arming anything
    d_full = ctx.reconcile_stats(ctx.read_stats(np.frombuffer(su.replies(zk, ctx.jute_requests(ZK_EXISTS)[0]), np.uint8)),
                                 SESSION)
    for i, (a, b) in enumerate(zip(d_sub.cls.tolist(), d_full.cls.tolist())):
        assert a == (b if i in dirty else (su.DUP if b == su.DUP else su.SAME)), i
    assert {paths[i] for i in dirty} == {paths[10], paths[12], paths[14]}
    ch_full = ctx.read_children(np.frombuffer(cu.replies(zk, ctx.children_requests()[0]), np.uint8))
    full_dirs = dirs_of(paths)
    assert ch_sub.n_unlisted == 0 and ch_sub.n_dirs == len(sub_dirs)
    lst_full = ch_full.listing()
    for k, dd in enumerate(sub_dirs):
        j = full_dirs.index(dd)
        a = lst_sub[int(ch_sub.child_off[k]):int(ch_sub.child_off[k + 1])]
        b = lst_full[int(ch_full.child_off[j]):int(ch_full.child_off[j + 1])]
        assert a == b
        assert ch_sub.cls[int(ch_sub.child_off[k]):int(ch_sub.child_off[k + 1])].tolist() == \
            ch_full.cls[int(ch_full.child_off[j]):int(ch_full.child_off[j + 1])].tolist()
    assert stale_sub == [ou.parent(paths[20]) + b"/stale-instance"]


def repair(ctx, zk):
    for op, kw in ((ZK_CREATE, dict(zk_flags=1)), (ZK_SETDATA, dict(observed_version=True)),
                   (ZK_REPLACE, dict(zk_flags=1, observed_version=True, group=5))):
        fb, fo, _ = ctx.reconcile_requests(op, xid_base=1000, **kw)
        assert set(zk.apply_frames(fb, fo, SESSION)) <= {ou.ZOK}
    fb, fo, _ = ctx.children_requests(ZK_DELETE, xid_base=3000)
    assert set(zk.apply_frames(fb, fo, SESSION)) <= {ou.ZOK}


def period(ctx, zk, xid):
    ev = ctx.read_events(np.frombuffer(zk.take_events(SESSION), np.uint8))
    fe = ctx.events_requests(ZK_EXISTS, xid_base=xid)[0]
    fc = ctx.events_requests(ZK_GETCHILDREN, xid_base=xid + 100000)[0]
    st = ctx.read_stats(serve(zk, fe))
    d = ctx.reconcile_stats(st, SESSION, zk_flags=1)
    ch = ctx.read_children(serve(zk, fc))
    return ev, st, d, ch


@pytest.mark.gpu
def test_the_watched_loop_end_to_end(ctx):
    paths, pays = batch(ctx, seed=21)
    zk = watched_model(paths, pays)
    arm(ctx, zk)
    drift(zk, paths, pays)
    ev, st, d, ch = period(ctx, zk, 10)
    assert d.n_create == 1 and d.n_update == 1 and d.n_replace == 1 and ch.n_stale == 1
    repair(ctx, zk)
    ev, st, d, ch = period(ctx, zk, 20)                                             # the repair's own events
    assert ev.n_events > 0 and st.n == ev.n_dirty_recs > 0
    assert d.n_create == d.n_update == d.n_replace == 0 and ch.n_stale == 0
    ev, st, d, ch = period(ctx, zk, 30)                                             # quiet
    assert ev.n_events == 0 and st.n == 0 and ch.n_dirs == 0
    first = {}
    for p, q in zip(paths, pays):
        first.setdefault(p, q)
    for p, q in first.items():
        assert zk.nodes[p].data == q and zk.nodes[p].owner == SESSION
    assert all(b"stale-instance" not in p for p in zk.nodes)
    # drift again after the repair: the re-armed watches see it
    zk.set_data(paths[12], b"x")
    ev, st, d, ch = period(ctx, zk, 40)
    assert st.n == 1 and d.n_update == 1


@pytest.mark.gpu
def test_a_million_records_with_ten_thousand_events(ctx):
    from registrar_b200 import synth
    b = synth.generate("config3", n=1_000_000, seed=5)
    ctx._last_batch = b
    got = ctx.register_batch(b)
    n = got.n
    rng = random.Random(9)
    picks = [rng.randrange(n) for _ in range(10_000)]
    paths = {i: got.path(i) for i in picks}
    s = b"".join(eu.notification(paths[i], rng.choice([2, 3])) for i in picks)
    a = np.frombuffer(s, np.uint8)
    g = ctx.read_events(a)
    m_first = {}
    for i in sorted(set(picks)):
        m_first.setdefault(paths[i], i)
    assert g.n_events == len(picks) and g.n_unmatched == 0
    # the subject is the first record with the path; DUP records of this batch are rare but exist
    for e, i in enumerate(picks):
        j = int(g.subject[e])
        assert j <= i and got.path(j) == paths[i]
    assert g.n_dirty_recs == len(set(int(x) for x in g.subject))
    g2 = ctx.read_events(a)                                                         # steady state: the same set
    assert g2.n_dirty_recs == g.n_dirty_recs
    fe = ctx.events_requests(ZK_EXISTS)[0]
    assert [p for _, _, p, _ in eu.parse_reads(fe.tobytes())] == [got.path(j) for j in sorted(set(int(x) for x in g.subject))]
