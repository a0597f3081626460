"""The replies to the library's write frames read back into each entry's outcome (regk_read_results), on the GPU: every
source and op against the restatement in results_util, groups 0 / 1 / 7 / 100, host and device streams at every start
phase, error codes in single frames and at the first, middle and last operation of a multi, a million config 3 creates,
a drifted registry repaired end to end in the ZooKeeper model, the state rules, every refusal, and the other calls'
results untouched.  CPU: the struct layout against the C compiler."""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import children_util as cu
import reconcile_owned_util as ou
import replies_util as ru
import results_util as su
from test_read_children import drifted, fleet_records, getchildren
from test_read_replies import getdata, model_of
from test_reconcile import _dev, run
from test_reconcile_owned import SESSION
from test_results_cpu import offsets

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZK_CREATE, ZK_DELETE, ZK_GETDATA, ZK_SETDATA, ZK_GETCHILDREN, ZK_REPLACE = 1, 2, 4, 5, 8, 256
RES_BATCH, RES_MKDIRP, RES_RECONCILE, RES_STALE = 1, 2, 3, 4
CODES = [-1, -2, -3, -4, -5, -6, -7, -8, -13, -14, -15, -100, -101, -102, -103, -108, -110, -111, -112, -113, -114, -115,
         -118, -119, -120, -121, -122, -123, -124, -125, -127]


def test_results_struct_layout_matches_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu ", sizeof(regk_results), offsetof(regk_results, consumed),
               offsetof(regk_results, flags), offsetof(regk_results, frame_err), offsetof(regk_results, cls),
               offsetof(regk_results, subject), offsetof(regk_results, aborted), offsetof(regk_results, kernel_ms),
               sizeof(regk_results_opts));
        printf("%u %u %u %u %u %u %u\n", REGK_RES_BATCH, REGK_RES_MKDIRP, REGK_RES_RECONCILE, REGK_RES_STALE, REGK_RES_DONE,
               REGK_RES_FAILED, REGK_RES_ABORTED);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    S = _native.CResults
    assert got == [C.sizeof(S), S.consumed.offset, S.flags.offset, S.frame_err.offset, S.cls.offset, S.subject.offset,
                   S.aborted.offset, S.kernel_ms.offset, C.sizeof(_native.CResultsOpts), _native.RES_BATCH,
                   _native.RES_MKDIRP, _native.RES_RECONCILE, _native.RES_STALE, _native.RES_DONE, _native.RES_FAILED,
                   _native.RES_ABORTED]
    assert "regk_read_results" in _native.EXPORTS


# ------------------------------------------------------------------------------------------------------------ GPU --

@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def check(ctx, stream, fr, source, op=None, subjects=None, start=0, phases=False):
    """read_results over host and device copies of `stream` against the restatement; returns the host-stream Results"""
    import torch
    subj = list(range(fr.entries)) if subjects is None else [int(x) for x in subjects]
    cases = [(stream, start)] + ([(b"\xab" * ph + stream, start + ph) for ph in range(1, 16)] if phases else [])
    for s, st in cases:
        want = su.read(s, fr, st)
        a = np.frombuffer(s, np.uint8)
        for dev in (False, True):
            got = ctx.read_results(torch.from_numpy(a.copy()).cuda() if dev else a, source, op, start=st)
            assert got.frame_err.tolist() == want["frame_err"]
            assert got.err.tolist() == want["err"] and got.cls.tolist() == want["cls"]
            assert got.version.tolist() == want["version"]
            assert got.subject.tolist() == subj
            assert got.failed.tolist() == [e for e, c in enumerate(want["cls"]) if c == su.FAILED]
            assert got.aborted.tolist() == [e for e, c in enumerate(want["cls"]) if c == su.ABORTED]
            assert (got.n_frames, got.n_entries, got.n_skipped, got.consumed) == (fr.frames, fr.entries, want["n_skipped"],
                                                                                  want["consumed"])
            assert got.n_done + got.n_failed + got.n_aborted == fr.entries
    raw = ctx.read_results(np.frombuffer(stream, np.uint8), source, op, start=start, device=True)
    want = su.read(stream, fr, start)
    assert _dev(ctx, raw.cls, fr.entries, np.uint8).tolist() == want["cls"]
    assert _dev(ctx, raw.subject, fr.entries, np.uint64).tolist() == subj
    assert _dev(ctx, raw.failed, int(raw.n_failed), np.uint64).tolist() == [e for e, c in enumerate(want["cls"]) if c == 1]
    return ctx.read_results(np.frombuffer(stream, np.uint8), source, op, start=start)


def copy_model(zk):
    z = ou.ZooKeeper()
    z.nodes = {p: n.copy() for p, n in zk.nodes.items()}
    return z


@pytest.mark.gpu
def test_batch_create_delete_setdata_in_groups(ctx):
    from registrar_b200.batch import RecordBatch
    paths, pays = run(ctx, RecordBatch.from_records(fleet_records(700, 9, seed=2)))
    base = model_of(paths, pays, skip=set(range(0, len(paths), 4)))
    for k in range(0, len(paths), 5):
        if paths[k] in base.nodes:
            base.set_data(paths[k], pays[k])                                        # version 1: BADVERSION at 0
    seen = set()
    for op in (ZK_CREATE, ZK_DELETE, ZK_SETDATA):
        for g in (0, 1, 7, 100):
            xb = 2 ** 31 - 50
            fb, fo, _ = ctx.jute_requests(op, xid_base=xb, zk_flags=1, version=-1 if op == ZK_DELETE else 0, group=g)
            zk = copy_model(base)
            nf = len(fo) - 1
            s = su.Server(zk, SESSION).replies(fb, fo, extra={0: su.ping(), 3: su.notification(b"/a"), nf: su.ping()},
                                               header_err={2: -4, nf - 1: -112})
            fr = su.Framing(op, paths, [len(p) for p in pays], xid_base=xb, group=g,
                            tol=su.NONODE if op == ZK_DELETE else 0)
            r = check(ctx, s, fr, RES_BATCH, phases=(op, g) == (ZK_CREATE, 7))
            seen |= set(r.cls.tolist())
            assert r.n_skipped == 2
    assert seen == {su.DONE, su.FAILED, su.ABORTED}
    # a getData framing leaves the record of the last write framing in force
    getdata(ctx, paths, 5)
    check(ctx, s, fr, RES_BATCH)


def rolled_back(xid, m, j, c):
    body = b"".join(su.mh(-1, False, x) + int(x).to_bytes(4, "big", signed=True)
                    for x in [0] * j + [c] + [-2] * (m - j - 1))
    return su._reply(xid, 0, body + su.mh(-1, True, -1))


@pytest.mark.gpu
def test_every_error_code_in_single_frames_and_multis(ctx):
    from registrar_b200.batch import RecordBatch
    n = 3 * 3 * len(CODES)
    paths, pays = run(ctx, RecordBatch.from_records(fleet_records(n, 4, seed=6)))
    for op in (ZK_DELETE, ZK_SETDATA):
        tol = su.NONODE if op == ZK_DELETE else 0
        ctx.jute_requests(op, xid_base=3, group=0)
        s = b"".join(su.error(3 + k, CODES[k % len(CODES)]) for k in range(n))
        r = check(ctx, s, su.Framing(op, paths, [len(p) for p in pays], 3, 0, tol), RES_BATCH)
        assert r.n_failed == n - (n // len(CODES) if tol else 0)
        ctx.jute_requests(op, xid_base=3, group=3)
        s = b"".join(rolled_back(3 + k, 3, k % 3, CODES[(k // 3) % len(CODES)]) for k in range(n // 3))
        r = check(ctx, s, su.Framing(op, paths, [len(p) for p in pays], 3, 3, tol), RES_BATCH)
        assert r.n_aborted == 2 * n // 3


@pytest.mark.gpu
def test_config3_million_creates(ctx):
    """the replies to a million single creates built on the device; 1 % NODEEXISTS"""
    import torch
    from registrar_b200 import synth
    n = 1_000_000
    res = ctx.register_batch(synth.generate("config3", n=n, seed=5))
    ctx.jute_requests(ZK_CREATE, xid_base=-2 ** 31 + 5, device=True)
    rng = np.random.default_rng(4)
    err = np.where(rng.random(n) < 0.01, su.NODEEXISTS, 0).astype(np.int32)
    stream = su.device_create_replies(res.path_bytes, res.path_off, -2 ** 31 + 5, err)
    got = ctx.read_results(stream, RES_BATCH)
    assert np.array_equal(got.err, err) and np.array_equal(got.cls, (err != 0).astype(np.uint8))
    assert np.array_equal(got.version, np.where(err == 0, 0, -1)) and got.consumed == stream.numel()
    assert np.array_equal(got.failed, np.flatnonzero(err).astype(np.uint64)) and got.n_aborted == 0
    del stream
    torch.cuda.empty_cache()


def _offsets(fb):
    return offsets(bytes(fb))


@pytest.mark.gpu
def test_end_to_end_repair_with_a_concurrent_writer(ctx):
    """the documented loop on a drifted registry; between the read and the repair another writer bumps versions,
    creates nodes and deletes nodes; the five sections' replies sit in one stream"""
    from registrar_b200.batch import RecordBatch
    paths, pays = run(ctx, RecordBatch.from_records(fleet_records(3000, 25, seed=9)))
    zk = drifted(paths, pays, random.Random(8))
    rng = random.Random(3)
    for p in rng.sample(paths, 300):                                                # UPDATE nodes: data drifted
        if p in zk.nodes:
            zk.nodes[p].data = b"drift"
    for p in rng.sample(paths, 100):                                                # REPLACE nodes: another session's
        if p in zk.nodes:
            zk.nodes[p].owner = 0x5EED
    srv = su.Server(zk, SESSION)
    for rounds in range(2):
        gd = getdata(ctx, paths, 11)
        fb = getchildren(ctx, paths, 11 + len(paths))
        s = ru.replies(zk, gd) + cu.replies(zk, fb)
        rep = ctx.read_replies(np.frombuffer(s, np.uint8))
        ch = ctx.read_children(np.frombuffer(s, np.uint8), start=rep.consumed)
        d = ctx.reconcile_owned(rep, session=SESSION, zk_flags=1)
        assert d.n_delete == 0
        expect = {}
        if rounds == 0:
            # the concurrent writer
            for i in d.update[::4]:
                zk.set_data(paths[int(i)], b"other")                                # BADVERSION
            for i in d.update[1::9]:
                zk.delete(paths[int(i)])                                            # NONODE
            for i in d.replace[::3]:
                zk.set_data(paths[int(i)], b"other")                                # BADVERSION in the replace
            for i in d.create[::5]:
                zk.create(paths[int(i)], b"first", 0x77)                            # NODEEXISTS
        sections = []
        xb = 100000
        stale = ch.stale_paths()
        fb, fo, _ = ctx.children_requests(ZK_DELETE, xid_base=xb)
        sections.append((fb, fo, RES_STALE, None, su.Framing(su.OP_DELETE, stale, xid_base=xb, tol=su.NONODE), ch.stale))
        dirs = ctx.mkdirp_dirs().dirs()
        fb, fo, _ = ctx.mkdirp_requests(xid_base=xb + 10000, zk_flags=0)
        sections.append((fb, fo, RES_MKDIRP, None, su.Framing(su.OP_CREATE, dirs, xid_base=xb + 10000,
                                                              tol=su.NODEEXISTS), None))
        for op, kw, lst, xo in ((ZK_CREATE, dict(zk_flags=1, group=7), d.create, 20000),
                                (ZK_SETDATA, dict(observed_version=True, group=3), d.update, 30000),
                                (ZK_REPLACE, dict(zk_flags=1, observed_version=True, group=5), d.replace, 40000)):
            fb, fo, _ = ctx.reconcile_requests(op, xid_base=xb + xo, **kw)
            sop = su.OP_REPLACE if op == ZK_REPLACE else op
            fr = su.Framing(sop, [paths[int(i)] for i in lst], [len(pays[int(i)]) for i in lst], xid_base=xb + xo,
                            group=kw["group"])
            sections.append((fb, fo, RES_RECONCILE, op, fr, lst))
        stream = b"".join(srv.replies(fb, fo, extra={0: su.ping()}) for fb, fo, _, _, _, _ in sections)
        start = 0
        for fb, fo, source, op, fr, subj in sections:
            got = check(ctx, stream, fr, source, op, subjects=subj, start=start)
            expect[(source, op)] = got
            start = got.consumed
        assert start == len(stream) or rounds == 1
        st = expect[(RES_STALE, None)]
        notempty = [stale[int(e)] for e in st.failed]
        assert notempty and all(p.endswith(b"/olddir") for p in notempty)
        assert set(st.err[st.failed.astype(np.int64)].tolist()) == {su.NOTEMPTY}
        if rounds == 0:
            assert sum(r.n_failed for r in expect.values()) > len(notempty)
            assert any(r.n_aborted for r in expect.values())
            upd = expect[(RES_RECONCILE, ZK_SETDATA)]
            assert {int(x) for x in upd.failed_subjects()} <= {int(i) for i in list(d.update[::4]) + list(d.update[1::9])}
        else:
            for (source, op), r in expect.items():
                if source != RES_STALE:
                    assert r.n_failed == r.n_aborted == 0, (source, op)
            want = {p: dd for p, dd in zip(paths, pays)}
            for p, dd in want.items():
                assert zk.nodes[p].data == dd and zk.nodes[p].owner == SESSION


@pytest.mark.gpu
def test_state_refusals_and_untouched_results(built):
    import torch
    from registrar_b200 import _native, synth
    from registrar_b200.batch import RecordBatch, Snapshot
    c = _native.Context(0)

    def refused(code, fn, *texts):
        with pytest.raises(_native.RegkError) as e:
            fn()
        assert e.value.code == code, e.value.message
        for t in texts:
            assert t in e.value.message, e.value.message

    try:
        ok = np.zeros(16, np.uint8)
        paths, pays = run(c, RecordBatch.from_records(fleet_records(800, 12, seed=12)))
        for src in (RES_BATCH, RES_MKDIRP, RES_STALE):
            refused(5, lambda: c.read_results(ok, src), "no write framing")
        refused(1, lambda: c.read_results(ok, 9), "source 9")
        refused(1, lambda: c.read_results(ok, RES_RECONCILE, ZK_GETDATA), "op 4")
        # results of the other calls
        zk = drifted(paths, pays, random.Random(1))
        gd = getdata(c, paths, 40)
        rep = c.read_replies(np.frombuffer(ru.replies(zk, gd), np.uint8))
        snap = rep.snapshot()
        fbc = getchildren(c, paths, 900)
        chs = c.read_children(np.frombuffer(cu.replies(zk, fbc), np.uint8))
        stale_before = chs.stale_paths()
        # a reconcile against a caller's snapshot holding nodes the batch does not produce: RECONCILE delete
        extra = [(b"/other/%d" % k, b"x") for k in range(30)]
        c.reconcile(Snapshot.from_nodes([(p, d) for p, d in zip(paths[:500], pays[:500])] + extra))
        fb, fo, _ = c.reconcile_requests(ZK_DELETE, xid_base=7, group=4)
        z2 = ou.ZooKeeper()
        z2.create(b"/other", b"", 0, ephemeral=False)
        for p, dd in extra[:20]:
            z2.create(p, dd, 0, ephemeral=False)
        s = su.Server(z2, SESSION).replies(fb, fo)
        dl = c.reconcile(Snapshot.from_nodes([(p, d) for p, d in zip(paths[:500], pays[:500])] + extra))
        refused(5, lambda: c.read_results(np.frombuffer(s, np.uint8), RES_RECONCILE, ZK_DELETE), "a reconcile ran")
        fb, fo, _ = c.reconcile_requests(ZK_DELETE, xid_base=7, group=4)
        r = check(c, s, su.Framing(su.OP_DELETE, [p for p, _ in extra], xid_base=7, group=4, tol=su.NONODE),
                  RES_RECONCILE, ZK_DELETE, subjects=dl.delete)
        assert r.subject.tolist() == list(range(500, 530))
        # a good create stream, and every refusal with its position
        xid = 5000
        fb, fo, _ = c.jute_requests(ZK_CREATE, xid_base=xid, group=3)
        fr = su.Framing(su.OP_CREATE, paths, xid_base=xid, group=3)
        good = su.Server(ou.ZooKeeper(), SESSION).replies(fb, fo)          # no parents: every multi rolls back NONODE
        good_ok = su.Server(model_of(paths, pays, skip=set(range(len(paths)))), SESSION).replies(fb, fo)
        check(c, good, fr, RES_BATCH)
        ends = offsets(good)
        k = 5
        at, nxt = ends[k], ends[k + 1]
        x = su.wrap(xid + k)
        fk = good[at:nxt]
        okk = offsets(good_ok)
        fk_ok = good_ok[okk[k]:okk[k + 1]]

        def with_frame(frame, base=good, e=ends):
            return base[:e[k]] + frame + base[e[k + 1]:]

        def flip(frame, i):
            b = bytearray(frame)
            b[i] ^= 0x40
            return bytes(b)
        P0 = len(paths[3 * k])
        cases = [
            (good[:-5], "%d of %d replies complete" % (fr.frames - 1, fr.frames)),
            (with_frame(su.error(-3, su.NONODE)), "negative xid"),
            (with_frame(su.error(su.wrap(xid + k + 1), su.NONODE)), "out of order"),
            (with_frame(su.error(su.wrap(xid + 10 ** 6), su.NONODE)), "outside the framed"),
            (with_frame(b"\0\0\0\x14" + su.error(x, -4)[4:] + b"body"), "with a body"),
            (with_frame((len(fk)).to_bytes(4, "big") + fk[4:] + b"\0\0\0\0"), "fits neither"),
            (with_frame(flip(fk, 20 + 3)), "MultiHeader"),
            (with_frame(flip(fk, 20 + 12)), "two codes differ"),
            (with_frame(rolled_back(x, 3, 0, -101)[:20 + 13] + rolled_back(x, 3, 0, -101)[20:20 + 13] +
                        rolled_back(x, 3, 0, -101)[20 + 26:]), "order"),
            (with_frame(fk[:-9] + su.mh(-1, False, -1)), "closing"),
            (with_frame(rolled_back(x, 3, 0, 0)[:20] + rolled_back(x, 3, 2, 0)[20:]), "no nonzero"),
            (with_frame(flip(fk_ok, 20 + 9 + 4 + P0 - 1), good_ok, okk), "path echo"),
        ]
        for stream, text in cases:
            s = np.frombuffer(bytes(stream), np.uint8)
            with pytest.raises(su.Refused) as e:
                su.read(stream, fr)
            refused(1, lambda: c.read_results(s, RES_BATCH), text, "byte %d" % e.value.pos, "xid %d" % su.wrap(xid + e.value.k))
            refused(1, lambda: c.read_results(torch.from_numpy(s.copy()).cuda(), RES_BATCH), text, "byte %d" % e.value.pos)
        # a setData Stat whose dataLength differs from the framed payload
        fb, fo, _ = c.jute_requests(ZK_SETDATA, xid_base=xid)
        sd = su.Server(model_of(paths, pays), SESSION).replies(fb, fo)
        e0 = offsets(sd)
        bad = sd[:e0[2] + 20 + 52] + b"\0\0\0\0" + sd[e0[2] + 20 + 56:]
        refused(1, lambda: c.read_results(np.frombuffer(bad, np.uint8), RES_BATCH), "dataLength", "byte %d" % (e0[2] + 72))
        refused(1, lambda: c.read_results(np.zeros(0, np.uint8), RES_BATCH), "0 of %d replies complete" % len(paths))
        refused(1, lambda: c.read_results(ok, RES_BATCH, start=17), "past the stream")
        out, o = _native.CResults(), _native.CResultsOpts(RES_BATCH, 0, 0, 0)
        assert c._lib.regk_read_results(c._h, None, 5, 0, C.byref(o), C.byref(out)) == 1
        assert c._lib.regk_read_results(c._h, ok.ctypes.data_as(C.c_void_p), 16, 0, None, C.byref(out)) == 1
        dev = torch.zeros(len(sd) + 16, dtype=torch.uint8, device="cuda")
        refused(1, lambda: c.read_results(dev[1:1 + len(sd)], RES_BATCH), "misaligned")
        c.jute_requests(ZK_DELETE, xid_base=-5)
        refused(1, lambda: c.read_results(ok, RES_BATCH), "cover -1")
        # the other calls' results are untouched
        after = c.read_replies(np.frombuffer(ru.replies(zk, gd), np.uint8)).snapshot()
        for key in ("path_bytes", "path_off", "json_bytes", "json_off", "version", "owner"):
            assert np.array_equal(getattr(snap, key), getattr(after, key)), key
        assert c.read_children(np.frombuffer(cu.replies(zk, fbc), np.uint8)).stale_paths() == stale_before
        # the state each source framed
        c.mkdirp_dirs()
        c.mkdirp_requests()
        c.mkdirp_dirs()
        refused(5, lambda: c.read_results(ok, RES_MKDIRP), "regk_mkdirp_dirs ran")
        c.children_requests(ZK_DELETE)
        c.read_children(np.frombuffer(cu.replies(zk, fbc), np.uint8))
        refused(5, lambda: c.read_results(ok, RES_STALE), "regk_read_children ran")
        c.jute_requests(ZK_CREATE)
        run(c, synth.generate("config1"))
        refused(5, lambda: c.read_results(ok, RES_BATCH), "a batch finished")
    finally:
        c.close()
