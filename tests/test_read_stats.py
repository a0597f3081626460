"""The heartbeat by stat on the GPU: exists frames of a batch (regk_jute_requests with REGK_ZK_EXISTS), the reply stream
read into per-record Stats (regk_read_stats) and the batch classed from them (regk_reconcile_stats), every output against
the restatement in stats_util; the equivalence with the getData route wherever a Stat can see the difference; the
same-length limit and the mzxid baseline that lifts it; the loop of INTEGRATION.md §3 end to end in the ZooKeeper model."""
import ctypes as C
import random

import numpy as np
import pytest

import reconcile_owned_util as ou
import replies_util as ru
import results_util as rsu
import stats_util as su
from test_reconcile import _dev, run
from test_reconcile_owned import OLD, OTHER, SESSION, host_snapshot
from test_read_replies import model_of

ZK_CREATE, ZK_DELETE, ZK_EXISTS, ZK_GETDATA, ZK_SETDATA, ZK_REPLACE = 1, 2, 3, 4, 5, 256
RES_RECONCILE = 3


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def exists(ctx, paths, xid):
    """the batch's exists frames, checked against the restatement"""
    fb, fo, _ = ctx.jute_requests(ZK_EXISTS, xid_base=xid)
    assert fb.tobytes() == su.exists_frames(paths, xid)
    assert len(fo) == len(paths) + 1 and int(fo[-1]) == len(fb)
    return fb


FIELDS = (("err", "err"), ("version", "version"), ("ephemeral_owner", "owner"), ("data_length", "data_length"),
          ("mzxid", "mzxid"))


def check(ctx, paths, stream, xid, start=0):
    """read_stats over a host and a device copy of `stream` against the restatement, with both candidate kernels and
    with device outputs; returns the host-stream Stats"""
    import torch
    want = su.read(stream, xid, len(paths), start)
    a = np.frombuffer(stream, np.uint8)
    host = None
    for dev, shared in ((False, 0), (True, 0), (False, 1)):
        ctx.set_option("stats_cand_shared", shared)
        got = ctx.read_stats(torch.from_numpy(a.copy()).cuda() if dev else a, start=start)
        assert got.n == len(paths)
        for g, w in FIELDS:
            assert getattr(got, g).tolist() == want[w], g
        for k in ("n_found", "n_missing", "n_error", "n_skipped", "consumed"):
            assert getattr(got, k) == want[k], k
        assert got.n_found + got.n_missing + got.n_error == got.n
        host = host or got
    ctx.set_option("stats_cand_shared", 0)
    raw = ctx.read_stats(a, start=start, device=True)
    for (g, _), dt in zip(FIELDS, (np.int32, np.int32, np.int64, np.int32, np.int64)):
        assert np.array_equal(_dev(ctx, getattr(raw, g), host.n, dt), getattr(host, g)), g
    return ctx.read_stats(a, start=start)


def delta_equals(d, want):
    assert d.m == 0 and d.n_delete == 0 and d.obs_cls.size == 0 and d.delete.size == 0
    assert d.cls.tolist() == want["cls"] and d.match.tolist() == want["match"]
    for k in ("create", "update", "dup", "replace"):
        assert getattr(d, k).tolist() == want[k], k
    assert d.n_same + d.n_create + d.n_update + d.n_dup + d.n_replace == d.n


def repair_frames(ctx, groups=(0,)):
    """every create / setData / replace framing of the last reconcile, with observed versions where they exist"""
    out = []
    for g in groups:
        out.append(ctx.reconcile_requests(ZK_CREATE, xid_base=11, zk_flags=1, group=g)[0].tobytes())
        out.append(ctx.reconcile_requests(ZK_SETDATA, xid_base=2 ** 31 - 5, observed_version=True, group=g)[0].tobytes())
        out.append(ctx.reconcile_requests(ZK_SETDATA, xid_base=3, version=4, group=g)[0].tobytes())
        out.append(ctx.reconcile_requests(ZK_REPLACE, xid_base=-9, zk_flags=1, observed_version=True, group=g)[0].tobytes())
        fb, fo, _ = ctx.reconcile_requests(ZK_DELETE, observed_version=True, group=g)
        out.append((fb.tobytes(), len(fo)))
    return out


def registry(paths, pays, rng, same_length=False):
    """a registry in which every found node holds its record's bytes or a payload of another length (same_length=True:
    some hold other bytes of the same length): missing nodes, foreign and old-session ephemerals, persistent nodes,
    arbitrary versions"""
    import mkdirp_util
    zk = ou.ZooKeeper()
    firsts = {}
    for p, d in zip(paths, pays):
        firsts.setdefault(p, d)
    dirs = set()
    for p in firsts:
        dirs.update(mkdirp_util.ancestors(mkdirp_util.dir_of(p)))
    for dd in sorted(dirs, key=lambda x: x.count(b"/")):
        assert zk.create(dd, b"", 0, ephemeral=False) == ou.ZOK
    for k, (p, d) in enumerate(firsts.items()):
        mode = k % 10
        if mode == 0:
            continue
        owner = {1: OTHER, 2: OLD, 3: 0}.get(mode, SESSION)
        data = d + b" " if mode == 4 else d[:-3] if mode == 5 else d[:-1] + b"~" if mode == 6 and same_length else d
        assert zk.create(p, data, owner, ephemeral=owner != 0) == ou.ZOK
        for _ in range(rng.randrange(0, 3)):
            assert zk.set_data(p, data) == ou.ZOK
    return zk


@pytest.mark.gpu
def test_exists_frames(ctx):
    from registrar_b200 import _native, synth
    paths, _ = run(ctx, synth.generate("config1"))
    for xid in (1, 2 ** 31 - 3, -2 ** 31, -7):
        exists(ctx, paths, xid)
    with pytest.raises(_native.RegkError) as e:
        ctx.jute_requests(ZK_EXISTS, group=3)
    assert e.value.code == 1 and "multi" in e.value.message
    paths, pays = run(ctx, synth.generate("config5", n=50_000, seed=3))            # tiles over the staging budget
    exists(ctx, paths, 11)
    # an exists framing and a getData framing of one batch are both outstanding; the write framing's record stays
    paths, pays = run(ctx, synth.generate("config3", n=2000, seed=2))
    setdata = ctx.jute_requests(ZK_SETDATA, xid_base=900, group=7)
    fe = exists(ctx, paths, 50)
    fg = ctx.jute_requests(ZK_GETDATA, xid_base=5000)[0]
    assert fg.tobytes() == ru.getdata_frames(paths, 5000)
    zk = model_of(paths, pays)
    st = ctx.read_stats(np.frombuffer(su.replies(zk, fe), np.uint8))
    rep = ctx.read_replies(np.frombuffer(ru.replies(zk, fg), np.uint8))
    assert st.n_found == rep.n_found == len(paths)
    srv = rsu.Server(zk, SESSION)
    fo = setdata[1]
    res = ctx.read_results(np.frombuffer(srv.replies(setdata[0].tobytes(), [int(x) for x in fo]), np.uint8), 1)
    assert res.n_done == len(paths)
    # a paths-only batch has no payload lengths to class against
    ctx.register_batch(synth.generate("config1"), payloads=False)
    with pytest.raises(_native.RegkError) as e:
        ctx.jute_requests(ZK_EXISTS)
    assert e.value.code == 5


@pytest.mark.gpu
def test_found_missing_errors_and_skipped_frames(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=3000, seed=4))
    n = len(paths)
    fb = exists(ctx, paths, 100)
    zk = model_of(paths, pays)
    assert check(ctx, paths, su.replies(zk, fb), 100).n_found == n
    r = check(ctx, paths, su.replies(ou.ZooKeeper(), fb), 100)                      # exactly n error replies
    assert r.n_missing == n and r.consumed == 20 * n
    zk = model_of(paths, pays, skip=set(range(0, n, 3)))
    errors = {k: [-4, -102, -7, -112][k % 4] for k in range(1, n, 97)}
    r = check(ctx, paths, su.replies(zk, fb, errors=errors), 100)
    assert r.n_error == len(errors) and r.n_missing > 0 and r.n_found > 0
    # pings and notifications before, between and after; notification paths that embed well-formed stat replies with
    # in-range xids; trailing frames and a partial frame after the n-th reply are left alone
    inner = su.success(su.wrap(100 + 6), 3, 0, 5) + su.error(su.wrap(100 + 7), su.NONODE)
    extra = {0: su.notification(b"/a") + su.ping(), 5: su.ping(), 77: su.notification(b"/" + inner * 40), n: su.ping()}
    tail = su.success(su.wrap(100 + n), 1, 0, 5) + su.ping() + su.error(100, su.NONODE)[:9]
    s = su.replies(zk, fb, extra=extra, trailing=tail)
    r = check(ctx, paths, s, 100)
    assert r.n_skipped == 4 and r.consumed == len(s) - len(tail) - len(su.ping())
    # every start phase, after another section of the stream
    for phase in range(16):
        front = ru.ping() * 3 + bytes(range(phase))
        r = check(ctx, paths, front + s, 100, start=len(front))
        assert r.consumed == len(front) + len(s) - len(tail) - len(su.ping())


@pytest.mark.gpu
def test_one_record_and_wrapping_xids(ctx):
    from registrar_b200.batch import RecordBatch
    recs = [{"domain": b"d.example.com", "hostname": b"h%d" % i, "type": b"host", "address": b"10.0.0.%d" % i} for i in range(5)]
    paths, pays = run(ctx, RecordBatch.from_records(recs[:1]))
    fb = exists(ctx, paths, 2 ** 31 - 1)
    zk = model_of(paths, pays)
    r = check(ctx, paths, su.replies(zk, fb, extra={0: su.ping(), 1: su.ping()}), 2 ** 31 - 1)
    assert r.n_found == 1
    check(ctx, paths, su.replies(ou.ZooKeeper(), fb), 2 ** 31 - 1)
    paths, pays = run(ctx, RecordBatch.from_records(recs))
    fb = exists(ctx, paths, 2 ** 31 - 2)                                            # xids wrap inside the batch
    check(ctx, paths, su.replies(model_of(paths, pays, skip={2}), fb), 2 ** 31 - 2)


def both_routes(ctx, paths, pays, zk, xid=40, groups=(0,), known=None):
    """reconcile_stats and read_replies + reconcile_owned over the same registry: (stat delta, stat frames, getData
    delta, getData frames, Stats)"""
    fe = exists(ctx, paths, xid)
    fg = ctx.jute_requests(ZK_GETDATA, xid_base=xid + 7)[0]
    st = check(ctx, paths, su.replies(zk, fe), xid)
    d1 = ctx.reconcile_stats(st, session=SESSION, zk_flags=1, known_mzxid=known)
    f1 = repair_frames(ctx, groups)
    rep = ctx.read_replies(np.frombuffer(ru.replies(zk, fg), np.uint8))
    d2 = ctx.reconcile_owned(rep, session=SESSION, zk_flags=1)
    f2 = repair_frames(ctx, groups)
    return d1, f1, d2, f2, st


@pytest.mark.gpu
def test_equivalence_with_the_getdata_route(ctx):
    from registrar_b200 import synth
    from registrar_b200.batch import RecordBatch
    base = synth.generate("config3", n=3000, seed=21)
    recs = [base.record(i) for i in range(base.n)]
    recs += recs[5:400:7]                                                           # duplicate paths in the batch
    paths, pays = run(ctx, RecordBatch.from_records(recs, types=base.types))
    assert len(set(paths)) < len(paths)
    zk = registry(paths, pays, random.Random(4))
    d1, f1, d2, f2, st = both_routes(ctx, paths, pays, zk, groups=(0, 7, 100))
    want = su.classify(paths, pays, su.read(su.replies(zk, su.exists_frames(paths, 40)), 40, len(paths)), SESSION, 1)
    delta_equals(d1, want)
    assert d1.n_create and d1.n_update and d1.n_replace and d1.n_dup
    assert np.array_equal(d1.cls, d2.cls)
    for k in ("create", "update", "dup", "replace"):
        assert np.array_equal(getattr(d1, k), getattr(d2, k)), k
    assert f1 == f2                                                                 # byte-identical frames, versions included
    assert all(fb == b"" and nf == 1 for fb, nf in f1[4::5])                        # ZK_DELETE frames nothing
    # persistent nodes wanted (zk_flags 0): every ephemeral is REPLACE on both routes
    d1 = ctx.reconcile_stats(st, session=0, zk_flags=0)
    delta_equals(d1, su.classify(paths, pays, su.read(su.replies(zk, su.exists_frames(paths, 40)), 40, len(paths)), 0, 0))
    rep = ctx.read_replies(np.frombuffer(ru.replies(zk, ru.getdata_frames(paths, 47)), np.uint8))
    d2 = ctx.reconcile_owned(rep, session=0, zk_flags=0)
    assert np.array_equal(d1.cls, d2.cls) and d1.n_replace > 0


@pytest.mark.gpu
def test_same_length_drift_needs_the_baseline(ctx):
    import torch
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=2000, seed=9))
    n = len(paths)
    zk = model_of(paths, pays)
    fe = exists(ctx, paths, 10)
    base = check(ctx, paths, su.replies(zk, fe), 10)
    d = ctx.reconcile_stats(base, session=SESSION, known_mzxid=base.mzxid)          # a baseline equal to the current mzxid
    assert d.n_same == n
    drifted = list(range(3, n, 50))
    for i in drifted:
        assert zk.set_data(paths[i], pays[i][:-1] + b"~") == ou.ZOK                 # other bytes, the same length
    st = check(ctx, paths, su.replies(zk, fe), 10)
    assert ctx.reconcile_stats(st, session=SESSION).n_same == n                     # what a stat cannot see
    for known in (base.mzxid, torch.from_numpy(base.mzxid.copy()).cuda()):
        d = ctx.reconcile_stats(st, session=SESSION, known_mzxid=known)
        assert d.update.tolist() == drifted and d.n_same == n - len(drifted)
        delta_equals(d, su.classify(paths, pays, su.read(su.replies(zk, fe), 10, n), SESSION, 1, base.mzxid.tolist()))
    # the getData route sees the same records
    rep = ctx.read_replies(np.frombuffer(ru.replies(zk, ctx.jute_requests(ZK_GETDATA, xid_base=1)[0]), np.uint8))
    assert ctx.reconcile_owned(rep, session=SESSION).update.tolist() == drifted
    with pytest.raises(ValueError):
        ctx.reconcile_stats(st, session=SESSION, known_mzxid=base.mzxid[:-1])


@pytest.mark.gpu
def test_an_unknown_node_state_refuses_the_classification(ctx):
    from registrar_b200 import _native, synth
    paths, pays = run(ctx, synth.generate("config3", n=1500, seed=6))
    fe = exists(ctx, paths, 1)
    st = check(ctx, paths, su.replies(model_of(paths, pays), fe, errors={900: -112, 411: -4}), 1)
    assert st.n_error == 2 and st.err[411] == -4
    with pytest.raises(_native.RegkError) as e:
        ctx.reconcile_stats(st, session=SESSION)
    assert e.value.code == 5 and "record 411" in e.value.message and "-4" in e.value.message
    with pytest.raises(_native.RegkError) as e:                                    # and leaves no reconcile result
        ctx.reconcile_requests(ZK_CREATE)
    assert e.value.code == 5


def stat_round(ctx, paths, pays, zk, xid, known=None):
    fe = exists(ctx, paths, xid)
    st = check(ctx, paths, su.replies(zk, fe, extra={2: su.ping()}), xid)
    return st, ctx.reconcile_stats(st, session=SESSION, zk_flags=1, known_mzxid=known)


@pytest.mark.gpu
def test_the_heartbeat_loop_end_to_end(ctx):
    """register, drift the registry, round 0, a stat round, the repair applied to the model and read back with
    read_results, a new baseline, and a stat round with nothing to send"""
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=3000, seed=21))
    n = len(paths)
    zk = registry(paths, pays, random.Random(7), same_length=True)
    srv = rsu.Server(zk, SESSION)

    def round0(xid):
        """exists first, then getData, in one stream; the slice after the stats goes to read_replies"""
        fe = exists(ctx, paths, xid)
        fg = ctx.jute_requests(ZK_GETDATA, xid_base=xid + n)[0]
        stream = np.frombuffer(su.replies(zk, fe) + ru.replies(zk, fg), np.uint8)
        st = ctx.read_stats(stream)
        rep = ctx.read_replies(stream[st.consumed:])
        return st, ctx.reconcile_owned(rep, session=SESSION, zk_flags=1)

    def repair():
        ctx.mkdirp_dirs()
        fb, fo, _ = ctx.mkdirp_requests(zk_flags=0)
        assert set(zk.apply_frames(fb, fo, SESSION)) <= {ou.ZOK, ou.NODEEXISTS}
        for op, kw in ((ZK_CREATE, dict(zk_flags=1, group=7)), (ZK_SETDATA, dict(observed_version=True, group=3)),
                       (ZK_REPLACE, dict(zk_flags=1, observed_version=True, group=5))):
            fb, fo, _ = ctx.reconcile_requests(op, xid_base=1000, **kw)
            s = srv.replies(fb.tobytes(), [int(x) for x in fo])
            res = ctx.read_results(np.frombuffer(s, np.uint8), RES_RECONCILE, op=op)
            assert res.n_failed == res.n_aborted == 0, op

    st, d = round0(2 ** 31 - 5000)
    assert d.n_create and d.n_update and d.n_replace
    same_len = int(d.n_update) - sum(1 for i in d.update.tolist() if len(zk.nodes[paths[i]].data) != len(pays[i]))
    assert same_len > 0                                                             # drift only the getData round sees
    repair()
    st, d = round0(5)                                                               # the new baseline
    assert d.n_same == n and st.n_found == n
    baseline = st.mzxid
    st, d = stat_round(ctx, paths, pays, zk, 77, baseline)
    assert d.n_same == n and d.n_create == d.n_update == d.n_replace == d.n_dup == 0
    for op in (ZK_CREATE, ZK_SETDATA, ZK_REPLACE, ZK_DELETE):
        assert ctx.reconcile_requests(op)[0].size == 0                              # nothing to send
    # the registry drifts again: a node lost, a foreign owner, a longer payload, a same-length rewrite
    zk.delete(paths[10])
    zk.delete(paths[11]), zk.create(paths[11], pays[11], OTHER)
    zk.set_data(paths[12], pays[12] + b"  ")
    zk.set_data(paths[13], pays[13][:-1] + b"~")
    st, d = stat_round(ctx, paths, pays, zk, 99, baseline)
    assert (d.create.tolist(), d.replace.tolist(), d.update.tolist()) == ([10], [11], [12, 13])
    repair()
    st, d = round0(300)
    assert d.n_same == n
    st, d = stat_round(ctx, paths, pays, zk, 400, st.mzxid)
    assert d.n_same == n


@pytest.mark.gpu
def test_refusals_and_state(built):
    import torch
    from registrar_b200 import _native, synth
    c = _native.Context(0)

    def refused(code, fn, *texts):
        with pytest.raises(_native.RegkError) as e:
            fn()
        assert e.value.code == code, e.value.message
        for t in texts:
            assert t in e.value.message, e.value.message

    try:
        paths, pays = run(c, synth.generate("config3", n=2000, seed=12))
        n = len(paths)
        ok = np.zeros(16, np.uint8)
        refused(5, lambda: c.read_stats(ok), "exists framing")                      # no framing yet
        refused(5, lambda: c.reconcile_stats(object(), session=SESSION), "regk_read_stats first")
        c.jute_requests(ZK_GETDATA)
        refused(5, lambda: c.read_stats(ok), "exists framing")                      # a getData framing is not one
        xid = 40
        fb = exists(c, paths, xid)
        zk = model_of(paths, pays)
        good = su.replies(zk, fb)
        ends, pos = [], 0
        while pos < len(good):
            pos += 4 + int.from_bytes(good[pos:pos + 4], "big")
            ends.append(pos)
        k = 700
        at, nxt = ends[k - 1], ends[k]
        x = su.wrap(xid + k)

        def with_frame(frame, lead=b""):
            return lead + good[:at] + frame + good[nxt:]

        ok_reply = su.success(x, 1, SESSION, 9)
        cases = [
            (good[:-5], "%d of %d replies complete" % (n - 1, n)),
            (good[:at] + b"\0\0\0\x0f" + b"\0" * 15 + good[at:], "below 16"),
            (with_frame(su.error(-3, su.NONODE)), "negative xid"),
            (with_frame(su.error(su.wrap(xid + k + 1), su.NONODE)), "out of order"),
            (with_frame(su.error(su.wrap(xid + k - 1), su.NONODE)), "out of order"),
            (with_frame(su.error(su.wrap(xid + n + 5), su.NONODE)), "outside the framed"),
            (with_frame(b"\0\0\0\x58" + ok_reply[4:] + b"data"), "not 84"),               # a getData-sized success
            (with_frame(ok_reply[:72] + b"\xff\xff\xff\xff" + ok_reply[76:]), "negative Stat.dataLength"),
            (with_frame(b"\0\0\0\x14" + su.error(x, -4)[4:] + b"body"), "with a body"),
        ]
        for stream, text in cases:
            for lead in (b"", su.ping() + b"abcde"):                                # the position counts from the stream's start
                s = np.frombuffer(lead + bytes(stream), np.uint8)
                refused(1, lambda: c.read_stats(s, start=len(lead)), text, "byte ", "xid ")
                refused(1, lambda: c.read_stats(torch.from_numpy(s.copy()).cuda(), start=len(lead)), text)
        lead = su.ping() + b"abcde"
        bad = np.frombuffer(with_frame(su.error(-3, su.NONODE), lead), np.uint8)
        refused(1, lambda: c.read_stats(bad, start=len(lead)), "byte %d" % (len(lead) + at), "record %d (xid %d)" % (k, x))
        refused(1, lambda: c.read_stats(np.zeros(0, np.uint8)), "0 of %d replies complete" % n)
        refused(1, lambda: c.read_stats(ok, start=17), "past the stream")
        # a fault after a refused read leaves no stats to class
        refused(5, lambda: c.reconcile_stats(object(), session=SESSION), "regk_read_stats first")
        # NULL pointers and a misaligned device stream
        out = _native.CStats()
        g = np.frombuffer(good, np.uint8)
        assert c._lib.regk_read_stats(c._h, None, 5, 0, 0, C.byref(out)) == 1
        assert c._lib.regk_read_stats(c._h, g.ctypes.data_as(C.c_void_p), len(good), 0, 0, None) == 1
        assert c._lib.regk_reconcile_stats(c._h, None, 0, C.byref(_native.CDeltaOwned())) == 1
        dev = torch.zeros(len(good) + 16, dtype=torch.uint8, device="cuda")
        dev[1:1 + len(good)] = torch.from_numpy(g.copy()).cuda()
        refused(1, lambda: c.read_stats(dev[1:1 + len(good)]), "misaligned")
        with pytest.raises(ValueError):
            c.read_stats(np.zeros(4, np.int32))
        st = c.read_stats(g)
        assert st.n_found == n
        refused(1, lambda: c.reconcile_stats(st, session=SESSION, zk_flags=2), "zk_flags")
        refused(1, lambda: c.reconcile_stats(st, session=0, zk_flags=1), "session")
        # xid ranges that cover -1 or -2
        c.jute_requests(ZK_EXISTS, xid_base=-5)
        refused(1, lambda: c.read_stats(g), "cover -1")
        c.jute_requests(ZK_EXISTS, xid_base=-(n + 1))
        refused(1, lambda: c.read_stats(g), "cover -2")
        # reconcile, reconcile_owned and reconcile_stats in turn each leave a consistent state
        exists(c, paths, xid)
        st = c.read_stats(g)
        snap = host_snapshot([(p, d[:-1], 1, SESSION) for p, d in zip(paths[:500], pays[:500])])
        owned = c.reconcile_owned(snap, SESSION)
        owned_frames = c.reconcile_requests(ZK_SETDATA, observed_version=True)[0].tobytes()
        d = c.reconcile_stats(st, session=SESSION)
        assert d.n_same == n and c.reconcile_requests(ZK_DELETE)[0].size == 0 and c.reconcile_requests(ZK_SETDATA)[0].size == 0
        again = c.reconcile_owned(snap, SESSION)
        assert np.array_equal(again.cls, owned.cls) and again.n_delete == owned.n_delete == 0
        assert c.reconcile_requests(ZK_SETDATA, observed_version=True)[0].tobytes() == owned_frames
        plain = c.reconcile(snap)
        assert plain.n_update == 500
        refused(5, lambda: c.reconcile_requests(ZK_REPLACE), "regk_reconcile_owned")
        d = c.reconcile_stats(st, session=OTHER)
        assert d.n_replace == n and c.reconcile_requests(ZK_REPLACE, observed_version=True)[1].size == n + 1
        # a batch finished after the framing, after the read; a pending batch
        c.register_batch(synth.generate("config1"))
        refused(5, lambda: c.read_stats(g), "after the exists framing")
        refused(5, lambda: c.reconcile_stats(st, session=SESSION), "a batch finished after regk_read_stats")
        c.jute_requests(ZK_EXISTS, xid_base=1)
        c.set_option("async", 1)
        t = c.submit(synth.generate("config1", seed=3))
        refused(5, lambda: c.read_stats(g), "in flight")
        refused(5, lambda: c.reconcile_stats(st, session=SESSION), "in flight")
        c.collect(t)
        c.set_option("async", 0)
        refused(5, lambda: c.read_stats(g))
    finally:
        c.close()


def device_stat_replies(n, xid_base, version, owner, dlen, mzxid, missing):
    """the reply stream to every record of a batch, built on the device: record i's reply is a success carrying
    version[i], owner[i], dlen[i] and mzxid[i] (its Stat otherwise as replies_util.stat()), or NONODE where missing[i]"""
    import torch
    be = lambda v, w: np.ascontiguousarray(np.asarray(v).astype(">i%d" % w)).view(np.uint8).reshape(-1, w)
    flen = np.where(missing, 20, 88)
    off = np.zeros(n + 1, np.int64)
    np.cumsum(flen, out=off[1:])
    fr = np.zeros((n, 88), np.uint8)
    fr[:, 20:88] = np.frombuffer(ru.stat(), np.uint8)
    fr[:, 0:4] = be(flen - 4, 4)
    fr[:, 4:8] = be(np.array([su.wrap(xid_base + i) for i in range(n)], np.int64), 4)
    fr[:, 16:20] = be(np.where(missing, su.NONODE, 0), 4)
    fr[:, 28:36] = be(mzxid, 8)
    fr[:, 52:56] = be(version, 4)
    fr[:, 64:72] = be(owner, 8)
    fr[:, 72:76] = be(dlen, 4)
    keep = torch.from_numpy(np.arange(88)[None, :] < flen[:, None]).cuda()
    return torch.from_numpy(fr).cuda()[keep].contiguous(), int(off[-1])


@pytest.mark.gpu
def test_config3_at_scale(ctx):
    """one million records, the stream built on the device: 1 % NONODE, 10 % foreign owners, 1 % of another length, 1 %
    written since the baseline; counts and sampled records"""
    import torch
    from registrar_b200 import synth
    n = 1_000_000
    res = ctx.register_batch(synth.generate("config3", n=n, seed=5))
    xid = 2 ** 31 - 1000
    ctx.jute_requests(ZK_EXISTS, xid_base=xid, device=True)
    rng = np.random.default_rng(3)
    missing = rng.random(n) < 0.01
    version = rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)
    owner = np.where(rng.random(n) < 0.1, OTHER, SESSION).astype(np.int64)
    J = np.diff(res.json_off.astype(np.int64))
    dlen = np.where(rng.random(n) < 0.01, J + 1, J).astype(np.int32)
    known = rng.integers(1, 2 ** 62, n, dtype=np.int64)
    mzxid = np.where(rng.random(n) < 0.01, known + 1, known)
    stream, total = device_stat_replies(n, xid, version, owner, dlen, mzxid, missing)
    assert stream.numel() == total
    st = ctx.read_stats(stream)
    found = ~missing
    assert (st.n_found, st.n_missing, st.n_error, st.n_skipped, st.consumed) == (int(found.sum()), int(missing.sum()), 0, 0, total)
    assert np.array_equal(st.err, np.where(missing, su.NONODE, 0))
    for got, want in ((st.version, version), (st.ephemeral_owner, owner), (st.data_length, dlen), (st.mzxid, mzxid)):
        assert np.array_equal(got, np.where(found, want, 0))
    d = ctx.reconcile_stats(st, session=SESSION, known_mzxid=torch.from_numpy(known).cuda())
    foreign = found & (owner != SESSION)
    upd = found & ~foreign & ((dlen != J) | (mzxid != known))
    assert np.array_equal(d.create, np.flatnonzero(missing).astype(np.uint64))
    assert np.array_equal(d.replace, np.flatnonzero(foreign).astype(np.uint64))
    assert np.array_equal(d.update, np.flatnonzero(upd).astype(np.uint64))
    assert d.n_dup == 0 and d.n_same == n - int(missing.sum()) - int(foreign.sum()) - int(upd.sum())
    sample = rng.integers(0, n, 2000)
    assert np.array_equal(d.match[sample], np.where(missing[sample], su.NO_MATCH, sample).astype(np.uint64))
    # the setData frames carry each node's observed version
    fb, fo, _ = ctx.reconcile_requests(ZK_SETDATA, observed_version=True)
    for q in (0, len(fo) // 2, len(fo) - 2):
        frame = fb[int(fo[q]):int(fo[q + 1])].tobytes()
        assert frame[-4:] == int(version[int(d.update[q])]).to_bytes(4, "big", signed=True)
    del stream
    torch.cuda.empty_cache()
