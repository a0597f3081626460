"""getData frames of a batch (regk_jute_requests with REGK_ZK_GETDATA) and the reply stream read back into a snapshot
(regk_read_replies), on the GPU: every output against the restatement in replies_util, host and device streams, a
registry repaired end to end in the ZooKeeper model, every refusal, and the results of the other calls untouched.
CPU: the struct layout against the C compiler."""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import reconcile_owned_util as ou
import replies_util as ru
from test_reconcile import _dev, run
from test_reconcile_owned import OLD, OTHER, SESSION, _build_registry, fallback_case, host_snapshot, spilled_tiles

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZK_CREATE, ZK_DELETE, ZK_GETDATA, ZK_SETDATA, ZK_REPLACE = 1, 2, 4, 5, 256


def test_replies_struct_layout_matches_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu %zu ", sizeof(regk_replies), offsetof(regk_replies, consumed),
               offsetof(regk_replies, flags), offsetof(regk_replies, err), offsetof(regk_replies, node_rec),
               offsetof(regk_replies, snapshot), offsetof(regk_replies, version));
        printf("%zu %zu %u\n", offsetof(regk_replies, ephemeral_owner), offsetof(regk_replies, kernel_ms), REGK_ZK_GETDATA);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    R = _native.CReplies
    assert got == [C.sizeof(R), R.consumed.offset, R.flags.offset, R.err.offset, R.node_rec.offset, R.snapshot.offset,
                   R.version.offset, R.ephemeral_owner.offset, R.kernel_ms.offset, _native.ZK_GETDATA]
    assert "regk_read_replies" in _native.EXPORTS


# ------------------------------------------------------------------------------------------------------------ GPU --

@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def getdata(ctx, paths, xid):
    """the batch's getData frames, checked against the restatement"""
    fb, fo, _ = ctx.jute_requests(ZK_GETDATA, xid_base=xid)
    assert fb.tobytes() == ru.getdata_frames(paths, xid)
    assert len(fo) == len(paths) + 1 and int(fo[-1]) == len(fb)
    return fb


def check(ctx, paths, stream, xid):
    """read_replies over a host and a device copy of `stream` against the restatement; returns the host-stream Replies"""
    import torch
    want = ru.read(stream, xid, len(paths))
    rec, nodes = ru.snapshot_nodes(paths, want)
    for dev in (False, True):
        a = np.frombuffer(stream, np.uint8)
        got = ctx.read_replies(torch.from_numpy(a.copy()).cuda() if dev else a)
        assert got.n == len(paths) and got.m == len(nodes)
        assert got.err.tolist() == want["err"]
        assert got.node_rec.tolist() == rec
        for k in ("n_found", "n_missing", "n_error", "n_skipped", "consumed"):
            assert getattr(got, k) == want[k], k
        assert got.n_found + got.n_missing + got.n_error == got.n
        s = got.snapshot()
        want_s = host_snapshot(nodes) if nodes else None
        if nodes:
            for k in ("path_bytes", "path_off", "json_bytes", "json_off", "version", "owner"):
                assert np.array_equal(getattr(s, k), getattr(want_s, k)), k
        else:
            assert s.path_off.tolist() == [0] and s.json_off.tolist() == [0]
        if not dev:
            host = got
    raw = ctx.read_replies(np.frombuffer(stream, np.uint8), device=True)
    assert np.array_equal(_dev(ctx, raw.err, host.n, np.int32), host.err)
    assert np.array_equal(_dev(ctx, raw.node_rec, host.m, np.uint64), host.node_rec)
    return ctx.read_replies(np.frombuffer(stream, np.uint8))


def model_of(paths, pays, owner=SESSION, skip=()):
    zk = ou.ZooKeeper()
    dirs = set()
    for p in paths:
        k = p.rindex(b"/")
        while k > 0:
            dirs.add(p[:k])
            k = p.rindex(b"/", 0, k)
    for d in sorted(dirs, key=lambda x: x.count(b"/")):
        zk.create(d, b"", 0, ephemeral=False)
    for i, (p, d) in enumerate(zip(paths, pays)):
        if i not in skip:
            zk.create(p, d, owner)
    return zk


@pytest.mark.gpu
def test_getdata_frames(ctx):
    from registrar_b200 import synth
    from registrar_b200.batch import RecordBatch
    paths, _ = run(ctx, synth.generate("config1"))
    for xid in (1, 2 ** 31 - 3, -2 ** 31, -7):
        getdata(ctx, paths, xid)
    # skip mode: the kept records in order
    base = synth.generate("config3", n=4000, seed=8)
    recs = [base.record(i) for i in range(base.n)]
    for i in (0, 5, 1999, 3999):
        recs[i] = dict(recs[i], domain=recs[i]["domain"] + b"/x")
    paths, _ = run(ctx, RecordBatch.from_records(recs, types=base.types), skip_bad=True)
    assert len(paths) == 3996
    getdata(ctx, paths, 3)
    # tiles over the staging budget: config 5 and long alias paths
    paths, _ = run(ctx, synth.generate("config5", n=200_000, seed=3))
    getdata(ctx, paths, 11)
    paths, _, _ = fallback_case(ctx)
    assert 0 < spilled_tiles([len(p) for p in paths]) < (len(paths) + 63) // 64
    getdata(ctx, paths, 2 ** 31 - 100)
    # CREATE / DELETE / SETDATA frames are those of the restatement as before
    import reconcile_util as rcu
    paths, pays = run(ctx, synth.generate("config3", n=5000, seed=2))
    for op in (ZK_CREATE, ZK_DELETE, ZK_SETDATA):
        for g in (0, 7):
            fb, _, _ = ctx.jute_requests(op, xid_base=5, group=g, version=3, zk_flags=1)
            assert fb.tobytes() == rcu.frames(op, list(zip(paths, pays)), 5, g, zk_flags=1, version=3), (op, g)


@pytest.mark.gpu
def test_found_missing_errors_and_skipped_frames(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=3000, seed=4))
    fb = getdata(ctx, paths, 100)
    n = len(paths)
    zk = model_of(paths, pays)
    r = check(ctx, paths, ru.replies(zk, fb), 100)                                  # all found
    assert r.n_found == n and r.m == n
    r = check(ctx, paths, ru.replies(ou.ZooKeeper(), fb), 100)                      # all NONODE
    assert r.n_missing == n and r.m == 0
    zk = model_of(paths, pays, skip=set(range(0, n, 3)))                            # a mix, other errors
    errors = {k: [-4, -102, -7, -112][k % 4] for k in range(1, n, 97)}
    r = check(ctx, paths, ru.replies(zk, fb, errors=errors), 100)
    assert r.n_error == len(errors) and r.n_missing > 0 and r.n_found > 0
    # notifications and pings first, between replies and last; trailing frames and a partial frame after the n-th reply
    extra = {0: ru.notification(b"/a") + ru.ping(), 5: ru.ping(), 77: ru.notification(b"/q" * 300), n: ru.ping()}
    tail = ru.success(ru.wrap(100 + n), b"later") + ru.ping() + ru.error(100, ru.NONODE)[:9]
    s = ru.replies(zk, fb, extra=extra, trailing=tail)
    r = check(ctx, paths, s, 100)
    assert r.n_skipped == 4 and r.consumed == len(s) - len(tail) - len(ru.ping())


@pytest.mark.gpu
def test_null_empty_and_large_data(ctx):
    from registrar_b200.batch import RecordBatch
    recs = [{"domain": b"d%d.example.com" % (i % 3), "hostname": b"h%d" % i, "type": b"host", "address": b"10.0.0.%d" % i}
            for i in range(12)]
    paths, pays = run(ctx, RecordBatch.from_records(recs))
    fb = getdata(ctx, paths, -50)
    zk = model_of(paths, pays)
    for k in (0, 3, 4):
        zk.nodes[paths[k]].data = b""
    big = bytes(random.Random(1).getrandbits(8) for _ in range(1024 * 1024 - 200))
    zk.nodes[paths[7]].data = big                                                   # just under jute.maxbuffer
    zk.nodes[paths[8]].data = big[:65537]
    r = check(ctx, paths, ru.replies(zk, fb, null={0, 4}), -50)
    assert r.m == 12


@pytest.mark.gpu
def test_adversarial_data_and_duplicates(ctx):
    """node data holding copies of the frames that follow it; duplicate paths, one whose first reply is NONODE"""
    from registrar_b200.batch import RecordBatch
    recs = [{"domain": b"s%d.example.com" % (i % 5), "hostname": b"h%d" % (i % 40), "type": b"host",
             "address": b"10.1.%d.%d" % (i % 9, i % 11)} for i in range(200)]
    paths, pays = run(ctx, RecordBatch.from_records(recs))
    assert len(set(paths)) == 40
    xid = 9
    fb = getdata(ctx, paths, xid)
    zk = model_of(paths, pays)
    honest = ru.replies(zk, fb)
    for k, p in enumerate(paths[:40]):
        if p in zk.nodes:
            zk.nodes[p].data = honest[200 * k: 200 * k + 3000]                     # copies of well-formed reply frames
    errors = {k: ru.NONODE for k in range(0, 10)}                                   # first replies of some paths: NONODE
    s = ru.replies(zk, fb, errors=errors, extra={10: ru.ping()})
    r = check(ctx, paths, s, xid)
    assert r.m < r.n_found and len(set(paths)) < len(paths)
    # n = 1
    paths, pays = run(ctx, RecordBatch.from_records(recs[:1]))
    fb = getdata(ctx, paths, 2 ** 31 - 1)
    check(ctx, paths, ru.replies(model_of(paths, pays), fb, extra={0: ru.ping(), 1: ru.ping()}), 2 ** 31 - 1)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1_000_000, 10_000_000])
def test_config3_at_scale(ctx, n):
    """every record's reply built on the device; 1 % NONODE; the snapshot equals the batch's found records"""
    import torch
    from registrar_b200 import synth
    res = ctx.register_batch(synth.generate("config3", n=n, seed=5))
    ctx.jute_requests(ZK_GETDATA, xid_base=2 ** 31 - 1000, device=True)
    rng = np.random.default_rng(3)
    missing = rng.random(n) < 0.01
    version = rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)
    owner = np.where(rng.random(n) < 0.1, OTHER, SESSION).astype(np.int64)
    stream = ru.device_replies(res.json_bytes, res.json_off, 2 ** 31 - 1000, version, owner, missing)
    got = ctx.read_replies(stream)
    found = np.flatnonzero(~missing)
    assert np.array_equal(got.err, np.where(missing, ru.NONODE, 0))
    assert (got.n_found, got.n_missing, got.n_error, got.n_skipped) == (len(found), n - len(found), 0, 0)
    assert got.consumed == stream.numel()
    # config 3 paths are distinct: every found record is a node
    assert np.array_equal(got.node_rec, found.astype(np.uint64))
    s = got.snapshot()
    po, jo = res.path_off.astype(np.int64), res.json_off.astype(np.int64)
    assert np.array_equal(np.diff(s.path_off.astype(np.int64)), np.diff(po)[found])
    assert np.array_equal(np.diff(s.json_off.astype(np.int64)), np.diff(jo)[found])
    keep_p = np.repeat(~missing, np.diff(po))
    keep_j = np.repeat(~missing, np.diff(jo))
    assert np.array_equal(s.path_bytes, res.path_bytes[keep_p])
    assert np.array_equal(s.json_bytes, res.json_bytes[keep_j])
    assert np.array_equal(s.version, version[found]) and np.array_equal(s.owner, owner[found])
    d = ctx.reconcile_owned(got, session=SESSION, zk_flags=1)
    assert d.n_create == n - len(found) and d.n_replace == int((owner[found] != SESSION).sum()) and d.n_delete == 0
    assert d.n_update == 0
    del stream
    torch.cuda.empty_cache()


def _repair(ctx, zk):
    """the repair frames of the last reconcile_owned, applied to the model in the documented order"""
    fb, fo, _ = ctx.reconcile_requests(ZK_DELETE, observed_version=True)
    assert set(zk.apply_frames(fb, fo, SESSION)) <= {ou.ZOK}
    ctx.mkdirp_dirs()
    fb, fo, _ = ctx.mkdirp_requests(zk_flags=0)
    assert set(zk.apply_frames(fb, fo, SESSION)) <= {ou.ZOK, ou.NODEEXISTS}
    for op, kw in ((ZK_CREATE, dict(zk_flags=1, group=7)), (ZK_SETDATA, dict(observed_version=True, group=3)),
                   (ZK_REPLACE, dict(zk_flags=1, observed_version=True, group=5))):
        fb, fo, _ = ctx.reconcile_requests(op, **kw)
        assert set(zk.apply_frames(fb, fo, SESSION)) <= {ou.ZOK}, op


def _frames_of_repair(ctx):
    out = []
    for op, kw in ((ZK_DELETE, dict(observed_version=True)), (ZK_CREATE, dict(zk_flags=1, group=7)),
                   (ZK_SETDATA, dict(observed_version=True, group=3)), (ZK_REPLACE, dict(zk_flags=1, observed_version=True))):
        out.append(ctx.reconcile_requests(op, **kw)[0].tobytes())
    return out


@pytest.mark.gpu
def test_end_to_end_from_a_drifted_registry(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=3000, seed=21))
    zk, dirs = _build_registry(paths, pays, random.Random(4))
    assert any(n.owner == OTHER for n in zk.nodes.values()) and any(n.owner == OLD for n in zk.nodes.values())
    xid = 2 ** 31 - 500
    fb = getdata(ctx, paths, xid)
    stream = ru.replies(zk, fb, extra={3: ru.ping(), 100: ru.notification(paths[3])})
    rep = check(ctx, paths, stream, xid)
    assert rep.n_missing > 0 and rep.n_error == 0
    d = ctx.reconcile_owned(rep, session=SESSION, zk_flags=1)
    frames = _frames_of_repair(ctx)
    _, nodes = ru.snapshot_nodes(paths, ru.read(stream, xid, len(paths)))
    want = ctx.reconcile_owned(host_snapshot(nodes), SESSION, 1)
    for k in ("cls", "match", "obs_cls", "create", "update", "dup", "delete", "replace"):
        assert np.array_equal(getattr(d, k), getattr(want, k)), k
    assert _frames_of_repair(ctx) == frames
    assert d.n_create and d.n_update and d.n_replace and d.n_delete == 0
    ctx.reconcile_owned(rep, session=SESSION, zk_flags=1)
    _repair(ctx, zk)
    # the second round: fresh getData frames, replies from the repaired model
    fb = getdata(ctx, paths, 77)
    rep = check(ctx, paths, ru.replies(zk, fb), 77)
    assert rep.n_found == len(paths)
    again = ctx.reconcile_owned(rep, session=SESSION, zk_flags=1)
    dups = len(paths) - len(set(paths))
    assert again.n_same == again.n - dups and again.n_dup == dups
    assert again.n_create == again.n_update == again.n_delete == again.n_replace == 0


@pytest.mark.gpu
def test_refusals_and_untouched_results(built):
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
        ok = np.zeros(16, np.uint8)
        refused(5, lambda: c.read_replies(ok), "getData framing")                 # no framing yet
        refused(1, lambda: c.jute_requests(ZK_GETDATA, group=3), "multi")
        xid = 40
        fb = getdata(c, paths, xid)
        zk = model_of(paths, pays)
        good = ru.replies(zk, fb)
        n = len(paths)
        # results of the other calls, before any read
        raw = c.parent_dirs(device=True)
        before_par = (_dev(c, raw.parent_len, int(raw.n), np.uint32), _dev(c, raw.unique_first, int(raw.n_unique), np.uint64))
        dirs = c.mkdirp_dirs().dirs()
        mk_frames = c.mkdirp_requests()[0].tobytes()
        setdata = c.jute_requests(ZK_SETDATA, group=7)[0].tobytes()
        snap = host_snapshot([(p, d[:-1], 1, SESSION) for p, d in zip(paths[:500], pays[:500])])
        delta = c.reconcile_owned(snap, SESSION)
        rframes = c.reconcile_requests(ZK_SETDATA, observed_version=True)[0].tobytes()
        fb = getdata(c, paths, xid)                                                # framing again: the reads below use it
        # every refusal names the byte and the expected xid
        r = ru.read(good, xid, n)
        assert r["n_found"] == n
        ends, pos = [], 0
        b = good
        while pos < len(b):
            pos += 4 + int.from_bytes(b[pos:pos + 4], "big")
            ends.append(pos)
        k = 700
        at = ends[k - 1]                                                           # reply k starts here
        nxt = ends[k]

        def with_frame(frame):
            return np.frombuffer(good[:at] + frame + good[nxt:], np.uint8)

        x = ru.wrap(xid + k)
        abc, empty, ab = ru.success(x, b"abc"), ru.success(x, b""), ru.success(x, b"ab")
        cases = [
            (good[:-5], "%d of %d replies complete" % (n - 1, n)),
            (good[:at] + b"\0\0\0\x0f" + b"\0" * 15 + good[at:], "below 16"),
            (with_frame(ru.error(-3, ru.NONODE)), "negative xid"),
            (with_frame(ru.error(ru.wrap(xid + k + 1), ru.NONODE)), "out of order"),
            (with_frame(ru.error(ru.wrap(xid + k - 1), ru.NONODE)), "out of order"),
            (with_frame(ru.error(ru.wrap(xid + n + 5), ru.NONODE)), "outside the framed"),
            (with_frame(b"\0\0\0\x5a" + abc[4:-1]), "length disagrees"),                # len 90, D 3
            (with_frame(empty[:20] + b"\xff\xff\xff\xfe" + empty[24:]), "below -1"),       # D -2
            (with_frame(ab[:78] + b"\0\0\0\x03" + ab[82:]), "dataLength"),                  # Stat.dataLength 3, D 2
            (with_frame(b"\0\0\0\x14" + ru.error(x, -4)[4:] + b"body"), "with a body"),
        ]
        for stream, text in cases:
            s = np.frombuffer(bytes(stream), np.uint8)
            refused(1, lambda: c.read_replies(s), text, "byte ", "xid ")
            refused(1, lambda: c.read_replies(torch.from_numpy(s.copy()).cuda()), text)
        # the position and the expected xid are named
        refused(1, lambda: c.read_replies(with_frame(ru.error(-3, ru.NONODE))), "byte %d" % at, "record %d (xid %d)" % (k, x))
        refused(1, lambda: c.read_replies(np.zeros(0, np.uint8)), "0 of %d replies complete" % n)
        # NULL pointers and a misaligned device stream
        out = _native.CReplies()
        assert c._lib.regk_read_replies(c._h, None, 5, 0, C.byref(out)) == 1
        assert c._lib.regk_read_replies(c._h, np.frombuffer(good, np.uint8).ctypes.data_as(C.c_void_p), len(good), 0, None) == 1
        dev = torch.zeros(len(good) + 16, dtype=torch.uint8, device="cuda")
        dev[1:1 + len(good)] = torch.from_numpy(np.frombuffer(good, np.uint8).copy()).cuda()
        refused(1, lambda: c.read_replies(dev[1:1 + len(good)]), "misaligned")
        with pytest.raises(ValueError):
            c.read_replies(np.zeros(4, np.int32))
        # the read that works
        got = c.read_replies(np.frombuffer(good, np.uint8))
        assert got.n_found == n
        # xid ranges that cover -1 or -2
        c.jute_requests(ZK_GETDATA, xid_base=-5)
        refused(1, lambda: c.read_replies(np.frombuffer(good, np.uint8)), "cover -1")
        c.jute_requests(ZK_GETDATA, xid_base=-(n + 1))
        refused(1, lambda: c.read_replies(np.frombuffer(good, np.uint8)), "cover -2")
        c.jute_requests(ZK_GETDATA, xid_base=-1)
        refused(1, lambda: c.read_replies(np.frombuffer(good, np.uint8)), "cover -1")
        # the other calls' results are untouched by the reads
        after_par = (_dev(c, raw.parent_len, int(raw.n), np.uint32), _dev(c, raw.unique_first, int(raw.n_unique), np.uint64))
        assert all(np.array_equal(a, b) for a, b in zip(before_par, after_par))
        assert c.mkdirp_dirs().dirs() == dirs and c.mkdirp_requests()[0].tobytes() == mk_frames
        assert c.jute_requests(ZK_SETDATA, group=7)[0].tobytes() == setdata
        assert c.reconcile_requests(ZK_SETDATA, observed_version=True)[0].tobytes() == rframes
        again = c.reconcile_owned(snap, SESSION)
        assert np.array_equal(again.cls, delta.cls) and np.array_equal(again.update, delta.update)
        # a batch finished after the framing; a pending batch
        c.jute_requests(ZK_GETDATA, xid_base=xid)
        c.register_batch(synth.generate("config1"))
        refused(5, lambda: c.read_replies(np.frombuffer(good, np.uint8)), "after the getData framing")
        c.jute_requests(ZK_GETDATA, xid_base=1)
        c.set_option("async", 1)
        t = c.submit(synth.generate("config1", seed=3))
        refused(5, lambda: c.read_replies(np.frombuffer(good, np.uint8)), "in flight")
        c.collect(t)
        c.set_option("async", 0)
        refused(5, lambda: c.read_replies(np.frombuffer(good, np.uint8)))
    finally:
        c.close()
