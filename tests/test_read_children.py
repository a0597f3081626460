"""getChildren frames of a batch's service directories (regk_children_requests) and the reply stream read back into a
listing with every child classed KEEP or STALE (regk_read_children), on the GPU: every output against the restatement
in children_util, host and device streams at every start phase, the stale deletes, a registry cleaned end to end in the
ZooKeeper model, every refusal, and the results of the other calls untouched.  CPU: the struct layout against the C
compiler."""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import children_util as cu
import mkdirp_util
import reconcile_owned_util as ou
import reconcile_util as rcu
import replies_util as ru
from test_read_replies import _repair, getdata, model_of
from test_reconcile import _dev, run
from test_reconcile_owned import OTHER, SESSION

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZK_DELETE, ZK_GETDATA, ZK_SETDATA, ZK_GETCHILDREN = 2, 4, 5, 8


def test_children_struct_layout_matches_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu %zu %zu ", sizeof(regk_children), offsetof(regk_children, consumed),
               offsetof(regk_children, n_unlisted), offsetof(regk_children, flags), offsetof(regk_children, dir_rec),
               offsetof(regk_children, cls), offsetof(regk_children, unlisted), offsetof(regk_children, listing));
        printf("%zu %u %u\n", offsetof(regk_children, kernel_ms), REGK_ZK_GETCHILDREN, REGK_CHILD_STALE);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    S = _native.CChildren
    assert got == [C.sizeof(S), S.consumed.offset, S.n_unlisted.offset, S.flags.offset, S.dir_rec.offset, S.cls.offset,
                   S.unlisted.offset, S.listing.offset, S.kernel_ms.offset, _native.ZK_GETCHILDREN, _native.CHILD_STALE]
    assert {"regk_children_requests", "regk_read_children"} <= set(_native.EXPORTS)


# ------------------------------------------------------------------------------------------------------------ GPU --

@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def getchildren(ctx, paths, xid):
    """the batch's getChildren frames, checked against the restatement; returns the frames and the listed directories"""
    listed, _ = cu.dir_set(paths)
    fb, fo, _ = ctx.children_requests(ZK_GETCHILDREN, xid_base=xid)
    assert fb.tobytes() == cu.getchildren_frames([d for _, d in listed], xid)
    assert len(fo) == len(listed) + 1 and int(fo[-1]) == len(fb)
    return fb


def check(ctx, paths, stream, xid, start=0):
    """read_children over a host and a device copy of `stream` against the restatement; returns the host-stream Children"""
    import torch
    listed, unlisted = cu.dir_set(paths)
    want = cu.read(stream, xid, len(listed), start)
    listing, off, cls, stale = cu.classify(paths, want)
    a = np.frombuffer(stream, np.uint8)
    for dev in (False, True):
        got = ctx.read_children(torch.from_numpy(a.copy()).cuda() if dev else a, start=start)
        assert got.n_dirs == len(listed) and got.n_children == len(listing) and got.n_stale == len(stale)
        assert got.dir_rec.tolist() == [r for r, _ in listed]
        assert [paths[r][:n] for r, n in zip(got.dir_rec.tolist(), got.dir_len.tolist())] == [d for _, d in listed]
        assert got.err.tolist() == want["err"]
        assert got.child_off.tolist() == off
        assert got.cls.tolist() == cls and got.stale.tolist() == stale
        assert got.unlisted.tolist() == unlisted
        for k in ("n_found", "n_missing", "n_error", "n_skipped", "consumed"):
            assert getattr(got, k) == want[k], k
        assert got.listing() == listing
        assert got.stale_paths() == [listing[e] for e in stale]
    raw = ctx.read_children(a, start=start, device=True)
    d, m = int(raw.n_dirs), int(raw.n_children)
    assert _dev(ctx, raw.cls, m, np.uint8).tolist() == cls
    assert _dev(ctx, raw.child_off, d + 1, np.uint64).tolist() == off
    assert _dev(ctx, raw.stale, int(raw.n_stale), np.uint64).tolist() == stale
    return ctx.read_children(a, start=start)


def fleet_records(n, ndom, seed=1):
    rng = random.Random(seed)
    return [{"domain": b"svc%d.dc%d.example.com" % (i % ndom, i % 3), "hostname": b"h%d-%d" % (i, rng.randrange(1000)),
             "type": b"host", "address": b"10.0.%d.%d" % (i % 250, i % 7)} for i in range(n)]


def drifted(paths, pays, rng):
    """the batch's registry with stale children: other sessions' ephemerals, persistent leftovers, a stale directory
    with children, and a directory that does not exist yet"""
    zk = model_of(paths, pays, skip=set(range(0, len(paths), 11)))
    listed, _ = cu.dir_set(paths)
    for j, (_, d) in enumerate(listed):
        if j % 5 == 0:
            zk.create(d + b"/gone%d" % j, b"x", OTHER)                             # another session's ephemeral
        if j % 7 == 1:
            zk.create(d + b"/left%d" % j, b"y", 0, ephemeral=False)                # a persistent leftover
        if j % 13 == 2:
            zk.create(d + b"/olddir", b"", 0, ephemeral=False)                     # a stale directory with a child
            zk.create(d + b"/olddir/h", b"z", 0, ephemeral=False)
    return zk


@pytest.mark.gpu
def test_getchildren_frames_and_unlisted(ctx):
    from registrar_b200 import synth
    from registrar_b200.batch import RecordBatch
    paths, _ = run(ctx, synth.generate("config1"))
    for xid in (1, 2 ** 31 - 3, -2 ** 31, -7):
        getchildren(ctx, paths, xid)
    # skip mode: the kept records
    base = synth.generate("config3", n=4000, seed=8)
    recs = [base.record(i) for i in range(base.n)]
    for i in (0, 5, 1999, 3999):
        recs[i] = dict(recs[i], domain=recs[i]["domain"] + b"/x")
    paths, _ = run(ctx, RecordBatch.from_records(recs, types=base.types), skip_bad=True)
    assert len(paths) == 3996
    getchildren(ctx, paths, 3)
    # "/" and directories ZooKeeper rejects are not listed: their first records come back in unlisted
    doms = [b"a.b", b"", b"x\x01.y.z", b"a.b", b"q.x\x7f.z", b"", b"c.d", b"w\x1f"]
    recs = [{"domain": d, "hostname": b"h%d" % i, "type": b"host", "address": b"1.1.1.1"} for i, d in enumerate(doms)]
    paths, pays = run(ctx, RecordBatch.from_records(recs))
    fb = getchildren(ctx, paths, 9)
    listed, unlisted = cu.dir_set(paths)
    assert len(listed) == 2 and unlisted == [1, 2, 4, 7]
    got = check(ctx, paths, cu.replies(model_of(paths, pays), fb), 9)
    assert got.n_unlisted == 4 and got.n_stale == 0


@pytest.mark.gpu
def test_listing_classes_errors_and_skipped_frames(ctx):
    from registrar_b200.batch import RecordBatch
    paths, pays = run(ctx, RecordBatch.from_records(fleet_records(3000, 40)))
    xid = 100
    fb = getchildren(ctx, paths, xid)
    zk = drifted(paths, pays, random.Random(3))
    d = len(cu.dir_set(paths)[0])
    r = check(ctx, paths, cu.replies(zk, fb), xid)
    assert r.n_stale > 0 and r.n_found == d
    # NONODE, other errors, null vectors, empty directories, notifications and pings, a stream that goes on
    for k in (3, 8):
        for p in [p for p in zk.nodes if p.startswith(cu.parse_getchildren(fb)[k][1] + b"/")]:
            del zk.nodes[p]
    zk.nodes.pop(cu.parse_getchildren(fb)[4][1])
    extra = {0: cu.notification(b"/a") + cu.ping(), 5: cu.ping(), 17: cu.notification(b"/q" * 300), d: cu.ping()}
    tail = cu.success(cu.wrap(xid + d), [b"later"]) + cu.ping() + cu.error(xid, cu.NONODE)[:9]
    s = cu.replies(zk, fb, errors={6: -4, 11: -102}, null={3}, extra=extra, trailing=tail)
    r = check(ctx, paths, s, xid)
    assert r.n_missing == 1 and r.n_error == 2 and r.n_skipped == 4 and r.consumed == len(s) - len(tail) - len(cu.ping())
    assert r.child_off[4] == r.child_off[5] and r.child_off[3] == r.child_off[4]


@pytest.mark.gpu
def test_start_at_every_phase(ctx):
    """the getData replies and the getChildren replies in one stream: read_children(start=consumed)"""
    from registrar_b200.batch import RecordBatch
    paths, pays = run(ctx, RecordBatch.from_records(fleet_records(500, 9, seed=2)))
    zk = drifted(paths, pays, random.Random(5))
    gd = getdata(ctx, paths, 7)
    fb = getchildren(ctx, paths, 7 + len(paths))
    ch = cu.replies(zk, fb, extra={1: cu.ping()})
    for phase in range(16):
        s = ru.replies(zk, gd, extra={0: b"" if phase == 0 else ru.notification(b"/" + b"p" * (phase + 2))}) + ch
        pre = len(s) - len(ch)
        rep = ctx.read_replies(np.frombuffer(s, np.uint8))
        assert rep.consumed == pre
        check(ctx, paths, s, 7 + len(paths), start=rep.consumed)
    check(ctx, paths, b"\xee" * 5 + ch, 7 + len(paths), start=5)


@pytest.mark.gpu
def test_one_directory_with_100k_children(ctx):
    from registrar_b200.batch import RecordBatch
    recs = [{"domain": b"big.example.com", "hostname": b"i%06d" % i, "type": b"host", "address": b"10.0.0.1"}
            for i in range(100_000)]
    paths, pays = run(ctx, RecordBatch.from_records(recs))
    fb = getchildren(ctx, paths, 1)
    names = [b"i%06d" % i for i in range(100_000)] + [b"stale%d" % i for i in range(3000)]
    random.Random(1).shuffle(names)
    s = cu.success(1, names)
    assert len(s) > 1_000_000
    r = check(ctx, paths, s, 1)
    assert r.n_children == 103_000 and r.n_stale == 3000


@pytest.mark.gpu
def test_a_million_directories_with_one_child_each(ctx):
    from registrar_b200 import synth
    import struct
    paths, _ = run(ctx, synth.generate("config3", n=1_000_000, seed=6))
    listed, _ = cu.dir_set(paths)
    assert len(listed) > 900_000
    fb, fo, _ = ctx.children_requests(ZK_GETCHILDREN, xid_base=1000)
    assert len(fo) == len(listed) + 1
    parts = []
    for k, (r, d) in enumerate(listed):
        name = paths[r][len(d) + 1:] if k % 97 else b"stale"
        parts.append(struct.pack(">iiqiii", 24 + len(name), cu.wrap(1000 + k), 0, 0, 1, len(name)) + name)
    s = b"".join(parts)
    got = ctx.read_children(np.frombuffer(s, np.uint8))
    assert got.n_dirs == len(listed) and got.n_children == len(listed) and got.consumed == len(s)
    want_stale = [k for k in range(len(listed)) if k % 97 == 0]
    assert got.stale.tolist() == want_stale and got.child_off.tolist() == list(range(len(listed) + 1))
    lst = got.listing()
    assert lst[1] == paths[listed[1][0]] and lst[0] == listed[0][1] + b"/stale"


@pytest.mark.gpu
def test_stale_delete_frames(ctx):
    from registrar_b200.batch import RecordBatch
    paths, pays = run(ctx, RecordBatch.from_records(fleet_records(2000, 30, seed=4)))
    fb = getchildren(ctx, paths, 1)
    r = check(ctx, paths, cu.replies(drifted(paths, pays, random.Random(2)), fb), 1)
    stale = r.stale_paths()
    assert len(stale) > 10
    for g in (0, 1, 7):
        for v in (-1, 12):
            got, fo, _ = ctx.children_requests(ZK_DELETE, xid_base=2 ** 31 - 2, version=v, group=g)
            assert got.tobytes() == rcu.frames(ZK_DELETE, [(p, b"") for p in stale], 2 ** 31 - 2, g, version=v), (g, v)
            assert len(fo) == (len(stale) + max(g, 1) - 1) // max(g, 1) + 1


@pytest.mark.gpu
def test_end_to_end_cleanup(ctx):
    from registrar_b200.batch import RecordBatch
    paths, pays = run(ctx, RecordBatch.from_records(fleet_records(3000, 25, seed=9)))
    zk = drifted(paths, pays, random.Random(8))
    for rounds in range(2):
        gd = getdata(ctx, paths, 11)
        fb = getchildren(ctx, paths, 11 + len(paths))
        s = ru.replies(zk, gd, extra={5: ru.ping()}) + cu.replies(zk, fb, extra={2: cu.notification(b"/x")})
        rep = ctx.read_replies(np.frombuffer(s, np.uint8))
        ch = check(ctx, paths, s, 11 + len(paths), start=rep.consumed)
        d = ctx.reconcile_owned(rep, session=SESSION, zk_flags=1)
        fb, fo, _ = ctx.children_requests(ZK_DELETE)
        res = zk.apply_frames(fb, fo, SESSION)
        if rounds == 0:
            assert ch.n_stale > 0 and d.n_create > 0
            olddirs = [p for p in ch.stale_paths() if p.endswith(b"/olddir")]
            assert olddirs and {res[k] for k, p in enumerate(ch.stale_paths()) if p in olddirs} == {ou.NOTEMPTY}
            assert {res[k] for k, p in enumerate(ch.stale_paths()) if p not in olddirs} == {ou.ZOK}
            _repair(ctx, zk)
            keep = cu.keep_set(paths)
            for _, dd in cu.dir_set(paths)[0]:
                kids = {dd + b"/" + n for n in cu.list_children(zk, dd)}
                assert kids <= keep | set(olddirs), dd
                assert {p for p in paths if mkdirp_util.dir_of(p) == dd} <= kids
        else:
            # the second round: only the NOTEMPTY directories remain stale, and reconcile has nothing to repair
            assert set(ch.stale_paths()) == set(olddirs) and set(res) <= {ou.NOTEMPTY}
            assert d.n_create == d.n_update == d.n_replace == d.n_delete == 0


@pytest.mark.gpu
def test_refusals_and_untouched_results(built):
    import torch
    from registrar_b200 import _native, synth
    from registrar_b200.batch import RecordBatch
    c = _native.Context(0)

    def refused(code, fn, *texts):
        with pytest.raises(_native.RegkError) as e:
            fn()
        assert e.value.code == code, e.value.message
        for t in texts:
            assert t in e.value.message, e.value.message

    try:
        ok = np.zeros(16, np.uint8)
        paths, pays = run(c, RecordBatch.from_records(fleet_records(1500, 20, seed=12)))
        refused(5, lambda: c.read_children(ok), "getChildren framing")
        refused(5, lambda: c.children_requests(ZK_DELETE), "stale list")
        refused(1, lambda: c.children_requests(ZK_GETCHILDREN, group=3), "multi")
        refused(1, lambda: c.children_requests(ZK_GETDATA), "not getChildren")
        refused(1, lambda: c.children_requests(ZK_SETDATA), "not getChildren")
        refused(1, lambda: c.jute_requests(ZK_GETCHILDREN), "op 8")
        # results of the other calls
        zk = drifted(paths, pays, random.Random(1))
        gd = getdata(c, paths, 40)
        rep = c.read_replies(np.frombuffer(ru.replies(zk, gd), np.uint8))
        snap = rep.snapshot()
        raw = c.parent_dirs(device=True)
        before_par = (_dev(c, raw.parent_len, int(raw.n), np.uint32), _dev(c, raw.unique_first, int(raw.n_unique), np.uint64))
        dirs = c.mkdirp_dirs().dirs()
        mk_frames = c.mkdirp_requests()[0].tobytes()
        c.reconcile_owned(rep, session=SESSION, zk_flags=1)
        rframes = c.reconcile_requests(ZK_SETDATA, observed_version=True)[0].tobytes()
        xid = 5000
        fb = getchildren(c, paths, xid)
        good = cu.replies(zk, fb)
        d = len(cu.dir_set(paths)[0])
        assert c.read_children(np.frombuffer(good, np.uint8)).n_stale > 0
        c.children_requests(ZK_DELETE, group=3)
        # every refusal names the byte and the expected xid
        ends, pos = [], 0
        while pos < len(good):
            pos += 4 + int.from_bytes(good[pos:pos + 4], "big")
            ends.append(pos)
        k = 7
        at, nxt = ends[k - 1], ends[k]
        x = cu.wrap(xid + k)

        def with_frame(frame):
            return good[:at] + frame + good[nxt:]
        cases = [
            (good[:-5], "%d of %d replies complete" % (d - 1, d), None),
            (with_frame(cu.error(-3, cu.NONODE)), "negative xid", at),
            (with_frame(cu.error(cu.wrap(xid + k + 1), cu.NONODE)), "out of order", at),
            (with_frame(cu.error(cu.wrap(xid + d + 5), cu.NONODE)), "outside the framed", at),
            (with_frame(cu.error(x, -4) + b""), None, None),
            (with_frame(b"\0\0\0\x14" + cu.error(x, -4)[4:] + b"body"), "with a body", at),
            (with_frame(cu.success(x, [b"a"])[:20] + b"\xff\xff\xff\xfe" + cu.success(x, [b"a"])[24:]), "below -1", at),
            (with_frame(cu.success(x, [b"ab", b"c"])[:20] + b"\0\0\0\x03" + cu.success(x, [b"ab", b"c"])[24:]),
             "too short", at),
            (with_frame(cu.success(x, [b"ab", b"c/d"])), "holding '/'", at + 24 + 6),
            (with_frame(cu.success(x, [b"ab", b"c\0d"])), "NUL", at + 24 + 6),
            (with_frame(cu.success(x, [b"..", b"c"])), "'.' or '..'", at + 24),
            (with_frame(cu.success(x, [b"ab", b""])), "empty name", at + 24 + 6),
            (with_frame(cu.success(x, [b"ab", b"cd"])[:20] + b"\0\0\0\x01" + cu.success(x, [b"ab", b"cd"])[24:]),
             "end before the frame", at + 24 + 6),
            (with_frame(b"\0\0\0\x1f" + cu.success(x, [b"ab", b"cd"])[4:-1]), "runs past", at + 24 + 6),
        ]
        for stream, text, where in cases:
            s = np.frombuffer(bytes(stream), np.uint8)
            if text is None:
                c.read_children(s)                                                  # an error reply is no refusal
                continue
            r = None
            try:
                r = cu.read(stream, xid, d)
            except cu.Refused as e:
                want_pos = e.pos
            assert r is None
            if where is not None:
                assert want_pos == where
            refused(1, lambda: c.read_children(s), text, "byte %d" % want_pos, "xid ")
            refused(1, lambda: c.read_children(torch.from_numpy(s.copy()).cuda()), text, "byte %d" % want_pos)
        refused(1, lambda: c.read_children(np.frombuffer(with_frame(cu.error(-3, 1)), np.uint8)),
                "directory %d (xid %d)" % (k, x))
        refused(1, lambda: c.read_children(np.zeros(0, np.uint8)), "0 of %d replies complete" % d)
        refused(1, lambda: c.read_children(ok, start=17), "past the stream")
        out = _native.CChildren()
        assert c._lib.regk_read_children(c._h, None, 5, 0, 0, C.byref(out)) == 1
        assert c._lib.regk_read_children(c._h, np.frombuffer(good, np.uint8).ctypes.data_as(C.c_void_p), len(good), 0, 0,
                                         None) == 1
        dev = torch.zeros(len(good) + 16, dtype=torch.uint8, device="cuda")
        dev[1:1 + len(good)] = torch.from_numpy(np.frombuffer(good, np.uint8).copy()).cuda()
        refused(1, lambda: c.read_children(dev[1:1 + len(good)]), "misaligned")
        # the other calls' results are untouched and still usable
        raw = c.parent_dirs(device=True)
        after = c.read_replies(np.frombuffer(ru.replies(zk, gd), np.uint8)).snapshot()
        for key in ("path_bytes", "path_off", "json_bytes", "json_off", "version", "owner"):
            assert np.array_equal(getattr(snap, key), getattr(after, key)), key
        assert np.array_equal(_dev(c, raw.parent_len, int(raw.n), np.uint32), before_par[0])
        assert np.array_equal(_dev(c, raw.unique_first, int(raw.n_unique), np.uint64), before_par[1])
        assert c.mkdirp_requests()[0].tobytes() == mk_frames and c.mkdirp_dirs().dirs() == dirs
        assert c.reconcile_requests(ZK_SETDATA, observed_version=True)[0].tobytes() == rframes
        # xid ranges that cover -1 or -2
        c.children_requests(ZK_GETCHILDREN, xid_base=-5)
        refused(1, lambda: c.read_children(np.frombuffer(good, np.uint8)), "cover -1")
        # a batch finished after the framing; alias, NO_PATH, empty and pending batches
        c.children_requests(ZK_GETCHILDREN, xid_base=1)
        run(c, synth.generate("config1"))
        refused(5, lambda: c.read_children(np.frombuffer(good, np.uint8)), "finished after")
        alias = RecordBatch.from_records([{"domain": b"a.b.c", "type": b"host", "address": b"1.1.1.1"}], alias=True)
        run(c, alias)
        refused(5, lambda: c.children_requests(ZK_GETCHILDREN), "alias")
        c.register_batch(synth.generate("config1"), paths=False)
        refused(5, lambda: c.children_requests(ZK_GETCHILDREN), "path stream")
        b1 = synth.generate("config1")
        run(c, RecordBatch.from_records([], types=b1.types))
        refused(5, lambda: c.children_requests(ZK_GETCHILDREN), "path stream")
        run(c, b1)
        c.set_option("async", 1)
        t = c.submit(b1)
        refused(5, lambda: c.children_requests(ZK_GETCHILDREN), "in flight")
        refused(5, lambda: c.read_children(ok), "in flight")
        c.collect(t)
        c.set_option("async", 0)
    finally:
        c.close()
