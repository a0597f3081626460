"""Every reply-stream reader (regk_read_replies, regk_read_stats with both candidate kernels, regk_read_children,
regk_read_results, regk_read_events with the SetWatches gate closed and open) against its sequential restatement, on
random and mutated streams and at the chain machinery's edges: a frame head at every phase of a 2 KiB span's last
block, stream lengths at and beside 2048 and 128 KiB multiples, candidate counts C of 1, 2, 3, 2^m and 2^m + 1 (both
all on the chain and mostly false), every `start` phase after a front that chains elsewhere, device streams viewed
inside a larger buffer whose bytes past the view would complete the last frame, and xid bases at the int32 edges.
Every case runs from a host array, from a device tensor and with device outputs.  CPU: the generators against the
restatements (every unmutated stream is accepted, and the planted phases, offsets and candidate counts are there)."""
import random
import re
import struct
import zlib

import numpy as np
import pytest

import children_util as cu
import events_util as eu
import reader_fuzz_util as fz
import reconcile_owned_util as ou
import reconcile_util as rcu
import replies_util as ru
import results_util as rsu
import setwatches_util as sw
import stats_util as su

ZK_CREATE, ZK_DELETE, ZK_EXISTS, ZK_GETDATA, ZK_SETDATA, ZK_GETCHILDREN = 1, 2, 3, 4, 5, 8
RES_BATCH = 1
SESSION = 0x1234_5678_9ABC_DEF0

# the reasons the library's refusals name, by each restatement's code (TRUNC: "the stream ends inside the frame", or
# "the stream ends before the reply ... is complete" where the chain stops)
HEAD = {1: "the stream ends", 2: "a frame length below 16 (no room for a ReplyHeader)",
        3: "a negative xid other than -1 (notification) or -2 (ping)", 4: "an xid outside the framed requests",
        5: "an error reply with a body"}
REPLY_REASON = {**HEAD, **{ru.SUCC_LEN: "a success frame whose length disagrees with its data length",
                             ru.NEG_DATA: "a data length below -1",
                             ru.STAT_LEN: "Stat.dataLength differs from the data the reply carries",
                             ru.ORDER: "a reply out of order, or for a record that already has one"}}
STATS_REASON = {**HEAD, **{su.SUCC_LEN: "a success frame whose length is not 84 (ReplyHeader + Stat)",
                             su.ORDER: "a reply out of order, or for a record that already has one",
                             su.NEG_DLEN: "a negative Stat.dataLength"}}
CHILDREN_REASON = {**HEAD, **{cu.SUCC_LEN: "a success frame too short for its count", cu.NEG_COUNT: "a child count below -1",
                                cu.ORDER: "a reply out of order, or for a directory that already has one",
                                cu.ENT_TRUNC: "an entry runs past the end of its frame",
                                cu.ENT_EMPTY: "an entry with an empty name", cu.NAME_SLASH: "a name holding '/'",
                                cu.NAME_NUL: "a name holding a NUL byte", cu.NAME_DOT: "a name that is '.' or '..'",
                                cu.ENT_END: "the entries end before the frame does"}}
RESULTS_REASON = {**HEAD, **{rsu.SUCC_LEN: "a success length that fits neither outcome of the frame",
                               rsu.ORDER: "a reply out of order, or for a frame that already has one",
                               rsu.OP_TYPE: "a MultiHeader of the wrong type, done flag or err",
                               rsu.PATH_ECHO: "a create path echo that differs from the framed path",
                               rsu.STAT_LEN: "Stat.dataLength differs from the framed data's length",
                               rsu.ERR_RESULT: "an ErrorResult whose two codes differ",
                               rsu.ERR_SEQ: "ErrorResults out of the 0 / failing code / -2 order",
                               rsu.CLOSE: "the multi's closing MultiHeader{-1, true, -1} is missing",
                               rsu.NO_FAILURE: "a rolled-back multi with no nonzero ErrorResult"}}
EVENTS_REASON = {eu.BAD_LEN: HEAD[2], eu.NEG_XID: "a negative xid other than -1 (notification) or -2 (ping), outside the "
                 "reply range", eu.XID_RANGE: "an xid outside the reply range",
                 eu.NOTE_LEN: "a notification whose length is not 28 + its path length",
                 eu.NEG_PATH: "a notification with a negative path length", eu.NOTE_ERR: "a notification with err != 0",
                 eu.TYPE: "a notification whose type is outside -1 .. 7", eu.PING_BODY: "a ping with a body",
                 sw.SW_BODY: "a SetWatches reply (xid -8) with a body", sw.SW_ERR: "a SetWatches reply (xid -8) with err != 0"}


def fleet(n, ndom=5, seed=1):
    rng = random.Random(seed)
    return [{"domain": b"svc%d.dc%d.example.com" % (i % ndom, i % 3), "hostname": b"h%d-%d" % (i, rng.randrange(1000)),
             "type": b"host", "address": b"10.0.%d.%d" % (i % 250, i % 7)} for i in range(n)]


def cpu_paths(n, ndom=5):
    """paths shaped as the library's for fleet(): for the generator self-test, which has no library to ask"""
    return [b"/com/example/dc%d/svc%d/h%d" % (i % 3, i % ndom, i) for i in range(n)], [b'{"a":%d}' % i for i in range(n)]


def model_of(paths, pays, skip=()):
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
            zk.create(p, d, SESSION)
    return zk


def _refused(text, pos, k):
    return ("refused", pos, text, k)


# ----------------------------------------------------------------------------------------------- the five readers --
# Each reader: the framing the library must produce (restated), an honest reply stream, the plausibility test, the
# restatement's outcome, and the library call with its outcome in the same form.

class Reader:
    has_start = True

    def __init__(self, paths, pays, xb):
        self.paths, self.pays, self.xb = list(paths), list(pays), xb
        self.zk = model_of(self.paths, self.pays, skip=set(range(0, len(self.paths), 5)))

    def frames(self, rng):
        return fz.split(self.honest(rng))


class Replies(Reader):
    name, has_start = "replies", False

    def framing(self):
        return ru.getdata_frames(self.paths, self.xb)

    def frame_on(self, ctx):
        return ctx.jute_requests(ZK_GETDATA, xid_base=self.xb)[0].tobytes()

    def honest(self, rng):
        n = len(self.paths)
        errs = {k: rng.choice([-4, -101, -102]) for k in rng.sample(range(n), min(n, 2))}
        return ru.replies(self.zk, self.framing(), errors=errs)

    def head(self, b, pos):
        return ru.plausible(b, pos, self.xb, len(self.paths))

    def want(self, b, start=0):
        try:
            r = ru.read(b, self.xb, len(self.paths))
        except ru.Refused as e:
            return _refused(REPLY_REASON[e.code], e.pos, e.k)
        rec, nodes = ru.snapshot_nodes(self.paths, r)
        from registrar_b200.batch import Snapshot
        s = Snapshot.from_nodes(nodes) if nodes else None
        snap = {k: getattr(s, k).tolist() for k in ("path_bytes", "path_off", "json_bytes", "json_off", "version",
                                                    "owner")} if s else None
        return ("ok", dict(err=r["err"], node_rec=rec, snap=snap,
                           counts=[r[k] for k in ("n_found", "n_missing", "n_error", "n_skipped", "consumed")]))

    def call(self, ctx, stream, start, device):
        return ctx.read_replies(stream, device=device)

    def outcome(self, ctx, g):
        s = g.snapshot()
        snap = {k: getattr(s, k).tolist() for k in ("path_bytes", "path_off", "json_bytes", "json_off", "version",
                                                    "owner")} if g.m else None
        if not g.m:
            assert s.path_off.tolist() == [0] and s.json_off.tolist() == [0]
        return ("ok", dict(err=g.err.tolist(), node_rec=g.node_rec.tolist(), snap=snap,
                           counts=[g.n_found, g.n_missing, g.n_error, g.n_skipped, g.consumed]))

    def outcome_dev(self, ctx, raw):
        n, m, s = int(raw.n), int(raw.m), raw.snapshot
        snap = dict(path_bytes=_dev(ctx, s.path_bytes, int(s.path_total), np.uint8).tolist(),
                    path_off=_dev(ctx, s.path_off, m + 1, np.uint64).tolist(),
                    json_bytes=_dev(ctx, s.json_bytes, int(s.json_total), np.uint8).tolist(),
                    json_off=_dev(ctx, s.json_off, m + 1, np.uint64).tolist(),
                    version=_dev(ctx, raw.version, m, np.int32).tolist(),
                    owner=_dev(ctx, raw.ephemeral_owner, m, np.int64).tolist()) if m else None
        return ("ok", dict(err=_dev(ctx, raw.err, n, np.int32).tolist(), node_rec=_dev(ctx, raw.node_rec, m, np.uint64).tolist(),
                           snap=snap, counts=[int(raw.n_found), int(raw.n_missing), int(raw.n_error), int(raw.n_skipped),
                                              int(raw.consumed)]))


class Stats(Reader):
    name = "stats"

    def __init__(self, paths, pays, xb, shared=0):
        super().__init__(paths, pays, xb)
        self.shared = shared
        self.name = "stats%d" % shared

    def framing(self):
        return su.exists_frames(self.paths, self.xb)

    def frame_on(self, ctx):
        ctx.set_option("stats_cand_shared", self.shared)
        return ctx.jute_requests(ZK_EXISTS, xid_base=self.xb)[0].tobytes()

    def honest(self, rng):
        n = len(self.paths)
        errs = {k: rng.choice([-4, -101, -102]) for k in rng.sample(range(n), min(n, 2))}
        return su.replies(self.zk, self.framing(), errors=errs)

    def head(self, b, pos):
        return su.plausible(b, pos, self.xb, len(self.paths))

    def want(self, b, start=0):
        try:
            r = su.read(b, self.xb, len(self.paths), start)
        except su.Refused as e:
            return _refused(STATS_REASON[e.code], e.pos, e.k)
        return ("ok", dict(arrays=[r[k] for k in ("err", "version", "owner", "data_length", "mzxid")],
                           counts=[r[k] for k in ("n_found", "n_missing", "n_error", "n_skipped", "consumed")]))

    def call(self, ctx, stream, start, device):
        assert ctx.get_option("stats_cand_shared") == self.shared
        return ctx.read_stats(stream, start=start, device=device)

    def outcome(self, ctx, g):
        return ("ok", dict(arrays=[a.tolist() for a in (g.err, g.version, g.ephemeral_owner, g.data_length, g.mzxid)],
                           counts=[g.n_found, g.n_missing, g.n_error, g.n_skipped, g.consumed]))

    def outcome_dev(self, ctx, raw):
        n = int(raw.n)
        got = [_dev(ctx, raw.err, n, np.int32), _dev(ctx, raw.version, n, np.int32),
               _dev(ctx, raw.ephemeral_owner, n, np.int64), _dev(ctx, raw.data_length, n, np.int32),
               _dev(ctx, raw.mzxid, n, np.int64)]
        return ("ok", dict(arrays=[a.tolist() for a in got], counts=[int(raw.n_found), int(raw.n_missing),
                                                                   int(raw.n_error), int(raw.n_skipped), int(raw.consumed)]))


class Children(Reader):
    name = "children"

    def __init__(self, paths, pays, xb, big=0):
        super().__init__(paths, pays, xb)
        self.dirs = [d for _, d in cu.dir_set(self.paths)[0]]
        self.big = big              # extra children of the first directory: a listing of that many more entries
        for j in range(big):
            self.zk.create(self.dirs[0] + b"/x%d" % j, b"", 0, ephemeral=False)
        for j, d in enumerate(self.dirs):
            if j % 3 == 1:
                self.zk.create(d + b"/gone%d" % j, b"x", 7)

    def framing(self):
        return cu.getchildren_frames(self.dirs, self.xb)

    def frame_on(self, ctx):
        return ctx.children_requests(ZK_GETCHILDREN, xid_base=self.xb)[0].tobytes()

    def honest(self, rng):
        d = len(self.dirs)
        return cu.replies(self.zk, self.framing(), errors={rng.randrange(d): -4} if d > 2 else None,
                          null=set(range(d)))

    def head(self, b, pos):
        return cu.plausible(b, pos, self.xb, len(self.dirs))

    def want(self, b, start=0):
        try:
            r = cu.read(b, self.xb, len(self.dirs), start)
        except cu.Refused as e:
            return _refused(CHILDREN_REASON[e.code], e.pos, e.k)
        listing, off, cls, stale = cu.classify(self.paths, r)
        return ("ok", dict(err=r["err"], off=off, cls=cls, stale=stale, listing=listing,
                           counts=[r[k] for k in ("n_found", "n_missing", "n_error", "n_skipped", "consumed")]))

    def call(self, ctx, stream, start, device):
        return ctx.read_children(stream, start=start, device=device)

    def outcome(self, ctx, g):
        return ("ok", dict(err=g.err.tolist(), off=g.child_off.tolist(), cls=g.cls.tolist(), stale=g.stale.tolist(),
                           listing=g.listing(), counts=[g.n_found, g.n_missing, g.n_error, g.n_skipped, g.consumed]))

    def outcome_dev(self, ctx, raw):
        d, m, s = int(raw.n_dirs), int(raw.n_children), raw.listing
        b = _dev(ctx, s.path_bytes, int(s.path_total), np.uint8).tobytes()
        off = _dev(ctx, s.path_off, m + 1, np.uint64).tolist()
        return ("ok", dict(err=_dev(ctx, raw.err, d, np.int32).tolist(), off=_dev(ctx, raw.child_off, d + 1, np.uint64).tolist(),
                           cls=_dev(ctx, raw.cls, m, np.uint8).tolist(),
                           stale=_dev(ctx, raw.stale, int(raw.n_stale), np.uint64).tolist(),
                           listing=[b[off[e]:off[e + 1]] for e in range(m)],
                           counts=[int(raw.n_found), int(raw.n_missing), int(raw.n_error), int(raw.n_skipped),
                                   int(raw.consumed)]))


class Results(Reader):
    def __init__(self, paths, pays, xb, op=ZK_CREATE, group=0):
        super().__init__(paths, pays, xb)
        self.op, self.group = op, group
        self.name = "results-%s-g%d" % ({ZK_CREATE: "create", ZK_DELETE: "delete", ZK_SETDATA: "setdata"}[op], group)
        self.version = -1 if op == ZK_DELETE else 0
        for k in range(1, len(self.paths), 6):
            if self.paths[k] in self.zk.nodes:
                self.zk.set_data(self.paths[k], self.pays[k])          # version 1: setData at 0 fails BADVERSION
        self.fr = rsu.Framing(op, self.paths, [len(p) for p in self.pays], xid_base=xb, group=group,
                              tol=rsu.NONODE if op == ZK_DELETE else 0)

    def framing(self):
        return rcu.frames(self.op, list(zip(self.paths, self.pays)), self.xb, self.group, zk_flags=1, version=self.version)

    def frame_on(self, ctx):
        return ctx.jute_requests(self.op, xid_base=self.xb, zk_flags=1, version=self.version, group=self.group)[0].tobytes()

    def honest(self, rng):
        fb = self.framing()
        fs = fz.split(fb)
        off = np.cumsum([0] + [len(f) for f in fs]).astype(np.uint64)
        zk = ou.ZooKeeper()
        zk.nodes = {p: n.copy() for p, n in self.zk.nodes.items()}
        return rsu.Server(zk, SESSION).replies(np.frombuffer(fb, np.uint8), off,
                                               header_err={rng.randrange(len(fs)): -4} if len(fs) > 2 else None)

    def head(self, b, pos):
        return rsu.plausible(b, pos, self.fr)

    def want(self, b, start=0):
        try:
            r = rsu.read(b, self.fr, start)
        except rsu.Refused as e:
            return _refused(RESULTS_REASON[e.code], e.pos, e.k)
        return ("ok", dict(arrays=[r["frame_err"], r["err"], r["cls"], r["version"]],
                           failed=[e for e, c in enumerate(r["cls"]) if c == rsu.FAILED],
                           aborted=[e for e, c in enumerate(r["cls"]) if c == rsu.ABORTED],
                           counts=[r["n_skipped"], r["consumed"]]))

    def call(self, ctx, stream, start, device):
        return ctx.read_results(stream, RES_BATCH, start=start, device=device)

    def outcome(self, ctx, g):
        assert g.subject.tolist() == list(range(self.fr.entries))
        assert (g.n_frames, g.n_entries) == (self.fr.frames, self.fr.entries)
        return ("ok", dict(arrays=[g.frame_err.tolist(), g.err.tolist(), g.cls.tolist(), g.version.tolist()],
                           failed=g.failed.tolist(), aborted=g.aborted.tolist(), counts=[g.n_skipped, g.consumed]))

    def outcome_dev(self, ctx, raw):
        f, e = int(raw.n_frames), int(raw.n_entries)
        assert (f, e) == (self.fr.frames, self.fr.entries)
        assert _dev(ctx, raw.subject, e, np.uint64).tolist() == list(range(e))
        return ("ok", dict(arrays=[_dev(ctx, raw.frame_err, f, np.int32).tolist(), _dev(ctx, raw.err, e, np.int32).tolist(),
                                   _dev(ctx, raw.cls, e, np.uint8).tolist(), _dev(ctx, raw.version, e, np.int32).tolist()],
                           failed=_dev(ctx, raw.failed, int(raw.n_failed), np.uint64).tolist(),
                           aborted=_dev(ctx, raw.aborted, int(raw.n_aborted), np.uint64).tolist(),
                           counts=[int(raw.n_skipped), int(raw.consumed)]))


class Events(Reader):
    """the session stream: notifications, pings and the replies to [xb, xb + nx); gate=True reads it after
    setwatches_requests() opened the SetWatches gate (xid -8 replies are frames then)"""

    def __init__(self, paths, pays, xb, nx=6, gate=False):
        super().__init__(paths, pays, xb)
        self.nx, self.gate = nx, gate
        self.name = "events-gate" if gate else "events"
        self.dirs = [d for _, d in cu.dir_set(self.paths)[0]]
        self.batch = None

    def framing(self):
        return b""

    def frame_on(self, ctx):
        return b""

    def honest(self, rng):
        parts = fz.noise(rng, self.paths + self.dirs, 30)
        for _ in range(4):
            if self.nx:
                x = ru.wrap(self.xb + rng.randrange(self.nx))
                parts.insert(rng.randrange(len(parts) + 1), cu.error(x, -101, zxid=rng.getrandbits(36)))
        parts += [eu.notification(d, eu.CHILDREN_CHANGED) for d in self.dirs[:3]]
        if self.gate:
            parts.insert(rng.randrange(len(parts) + 1), sw.reply(rng.getrandbits(36)))
        return b"".join(parts)

    def head(self, b, pos):
        return sw.head(b, pos, self.xb, self.nx, self.gate)

    def want(self, b, start=0):
        try:
            r = eu.read(b, self.xb, self.nx, start) if not self.gate else None
            m = sw.read(b, self.xb, self.nx, start, gate=self.gate)
        except eu.Refused as e:
            return _refused(EVENTS_REASON[e.code], e.pos, None)
        if self.gate:          # eu.read does not know xid -8: the events from the frames sw.read walks
            r = dict(events=[], n_pings=m["n_pings"], n_replies=m["n_replies"], consumed=m["consumed"],
                     partial=m["partial"])
            pos = start
            while pos < m["consumed"]:
                ln, xid = fz.be32(b, pos), fz.be32(b, pos + 4)
                if xid == eu.NOTIFY_XID:
                    typ, state, plen = struct.unpack_from(">iii", b, pos + 20)
                    r["events"].append((pos, typ, state, struct.unpack_from(">q", b, pos + 8)[0],
                                        bytes(b[pos + 32:pos + 32 + plen])))
                pos += 4 + ln
        mp = eu.Mapper(self.paths)
        subj, unmatched, other = mp.feed(r["events"])
        ev = r["events"]
        out = dict(pos=[e[0] for e in ev], type=[e[1] for e in ev], state=[e[2] for e in ev], zxid=[e[3] for e in ev],
                   subj=subj, counts=[len(ev), r["n_pings"], r["n_replies"], unmatched, other, r["consumed"],
                                      r["partial"], len(mp.dirty_recs), len(mp.dirty_dirs)], mark=m["mark"])
        if not self.gate:
            out["pending"] = ([self.paths[i] for i in mp.take()], [self.dirs[k] for k in mp.take(dirs=True)])
        return ("ok", out)

    def prepare(self, ctx):
        """a fresh batch generation: empty pending sets (and, with the gate, the gate opened)"""
        ctx.register_batch(self.batch)
        if self.gate:
            ctx.setwatches_requests()

    def call(self, ctx, stream, start, device):
        self.prepare(ctx)
        return ctx.read_events(stream, start=start, xid_base=self.xb, n_xids=self.nx, device=device)

    def outcome(self, ctx, g):
        out = dict(pos=g.pos.tolist(), type=g.type.tolist(), state=g.state.tolist(), zxid=g.zxid.tolist(),
                   subj=list(zip(g.subject_kind.tolist(), g.subject.tolist())),
                   counts=[g.n_events, g.n_pings, g.n_replies, g.n_unmatched, g.n_other, g.consumed, g.partial,
                           g.n_dirty_recs, g.n_dirty_dirs], mark=None)
        if self.gate:
            out["counts"][7:] = [None, None]        # setwatches_requests() made the whole batch pending
        else:
            out["pending"] = pending(ctx)
        return ("ok", out)

    def outcome_dev(self, ctx, raw):
        n = int(raw.n_events)
        out = dict(pos=_dev(ctx, raw.pos, n, np.uint64).tolist(), type=_dev(ctx, raw.type, n, np.int32).tolist(),
                   state=_dev(ctx, raw.state, n, np.int32).tolist(), zxid=_dev(ctx, raw.zxid, n, np.int64).tolist(),
                   subj=list(zip(_dev(ctx, raw.subject_kind, n, np.uint8).tolist(),
                                 _dev(ctx, raw.subject, n, np.uint64).tolist())),
                   counts=[n, int(raw.n_pings), int(raw.n_replies), int(raw.n_unmatched), int(raw.n_other),
                           int(raw.consumed), bool(raw.partial), int(raw.n_dirty_recs), int(raw.n_dirty_dirs)], mark=None)
        if self.gate:
            out["counts"][7:] = [None, None]
        else:
            out["pending"] = pending(ctx)
        return ("ok", out)


def pending(ctx):
    """the pending records' and directories' paths, as events_requests() frames them (the sets are then empty)"""
    recs = [p for _, _, p, _ in eu.parse_reads(ctx.events_requests(ZK_EXISTS, xid_base=1)[0].tobytes())]
    dirs = [p for _, _, p, _ in eu.parse_reads(ctx.events_requests(ZK_GETCHILDREN, xid_base=1)[0].tobytes())]
    return recs, dirs


def _dev(ctx, ptr, count, dtype):
    import ctypes as C
    out = np.zeros(count, dtype)
    if count:
        assert ctx._lib.regk_memcpy_d2h(ctx._h, out.ctypes.data_as(C.c_void_p), C.c_void_p(ptr), out.nbytes) == 0
    return out


def readers(paths, pays, xb=1):
    out = [Replies(paths, pays, xb), Stats(paths, pays, xb, 0), Stats(paths, pays, xb, 1), Children(paths, pays, xb)]
    for op, g in ((ZK_CREATE, 0), (ZK_DELETE, 1), (ZK_SETDATA, 7), (ZK_CREATE, 7)):
        out.append(Results(paths, pays, xb, op, g))
    out += [Events(paths, pays, xb), Events(paths, pays, xb, gate=True)]
    return out


NAMES = [r.name for r in readers(*cpu_paths(12))]
# candidate counts: 1, 2, 3, 2^m and 2^m + 1 up to m = 17, and either side of 8192 (64 tiles of 128 candidates, one
# super-tile of the chain passes' totals)
CS = sorted({1, 2, 3, 8191, 8192, 8193, 16383, 16385} | {2 ** m for m in range(1, 18)} | {2 ** m + 1 for m in range(1, 18)})


# ------------------------------------------------------------------------------------------------------ generators --

def honest_stream(rd, rng, noise=True, decoys=True, trailing=True):
    """the reader's honest replies with pings and notifications between them, notifications whose paths hold copies
    of this and the other readers' frames, and trailing frames (sometimes a partial one)"""
    frames = rd.frames(rng)
    extras = fz.noise(rng, rd.paths, rng.randrange(0, 6)) if noise else []
    if decoys and frames:
        copies = [ru.ping(), rng.choice(frames), su.success(rd.xb, 1, 2, 3), cu.success(rd.xb, [b"a", b"bb"]),
                  ru.success(rd.xb, b"data"), eu.notification(b"/n", 3)]
        rng.shuffle(copies)
        extras.append(fz.decoy(b"".join(copies)))
        extras.append(fz.decoy(b"".join(copies)[:rng.randrange(8, 64)]))
    b = b"".join(fz.interleave(frames, rng, extras))
    if trailing:
        t = b"".join(fz.noise(rng, rd.paths, rng.randrange(3)))
        t += fz.decoy(ru.ping() * 3 + (frames[0] if frames else b""))
        if rng.randrange(2):
            t = t[:rng.randrange(len(t) + 1)]
        b += t
    return b


def with_front(rd, b, start, rng):
    """the stream read from `start`, after `start` bytes that chain somewhere else"""
    return fz.long_front(start, rng) + b


def plain_frames(rd, rng):
    """the honest replies, no noise (for the events reader: a reply with a zxid, then notifications for three
    records)"""
    if not isinstance(rd, Events):
        return rd.frames(rng)
    return [cu.error(rd.xb, -101, zxid=0x5_0000_0000 + rng.getrandbits(20))] * (rd.nx > 0) + [
        eu.notification(p) for p in rd.paths[:3]]


def chain_to(rd, rng, C, false=False):
    """a stream whose candidate count from 0 is exactly C.  All on the chain: pings, then the plain frames (for the
    events reader as many of them as C leaves room for).  false=True: a notification whose path holds the pings (all
    off the chain), then the plain frames - or, where C is too small for that, the pings after a byte that is no
    frame head, so that no candidate is on the chain at all"""
    fr = plain_frames(rd, rng)
    while isinstance(rd, Events) and len(fr) > 1 and len(fz.cands(rd.head, b"".join(fr))) > C:
        fr.pop()
    base = b"".join(fr)
    c0 = len(fz.cands(rd.head, base))
    t = C - c0 - (1 if false else 0)
    if false and t < 1:
        out = b"\xff" + ru.ping() * C
    else:
        assert t >= 0, (rd.name, C, c0)
        out = (fz.decoy(ru.ping() * t) if false else ru.ping() * t) + base
    assert len(fz.cands(rd.head, out)) == C, (rd.name, C, false)
    return out


# --------------------------------------------------------------------------------------------------------- checks --

def expect_same(rd, want, got):
    assert want[0] == got[0], (rd.name, want, got)
    if want[0] == "refused":
        assert want[1:] == got[1:], (rd.name, want, got)
        return
    w, g = want[1], got[1]
    for k in w:
        if k == "mark" or g.get(k) is None:
            continue
        if k == "counts":
            assert [x for x, y in zip(w[k], g[k]) if y is not None] == [y for y in g[k] if y is not None], (rd.name, k)
        else:
            assert w[k] == g[k], (rd.name, k, w[k], g[k])


def outcome_of(rd, ctx, stream, start, device=False):
    from registrar_b200 import _native
    try:
        out = rd.call(ctx, stream, start, device)
    except _native.RegkError as e:
        m = re.search(r": byte (\d+): (.*)", e.message)
        assert m, e.message
        k = re.search(r"(?:expected the reply to|before the reply to) \w+ (\d+)", e.message)
        text = next((t for t in _reasons(rd) if m.group(2).startswith(t)), m.group(2))
        return ("refused", int(m.group(1)), text, int(k.group(1)) if k else None), None
    if device:
        return None, out
    return rd.outcome(ctx, out), out


def _reasons(rd):
    return {Replies: REPLY_REASON, Stats: STATS_REASON, Children: CHILDREN_REASON, Results: RESULTS_REASON,
            Events: EVENTS_REASON}[type(rd)].values()


def run_case(ctx, rd, b, start=0, view=b""):
    """the reader over `b` from `start` three ways - a host array, a device tensor viewing len(b) bytes of a buffer
    that continues with `view`, and device outputs - against the restatement; for the events reader also the zxid
    high-water mark"""
    import torch
    want = rd.want(b, start)
    a = np.frombuffer(b + view, np.uint8)[:len(b)]
    got, _ = outcome_of(rd, ctx, a, start)
    expect_same(rd, want, got)
    buf = torch.from_numpy(np.frombuffer(b + view + b"\0" * 16, np.uint8).copy()).cuda()
    got, _ = outcome_of(rd, ctx, buf[:len(b)], start)
    expect_same(rd, want, got)
    got, raw = outcome_of(rd, ctx, a, start, device=True)
    expect_same(rd, want, got if got is not None else rd.outcome_dev(ctx, raw))
    if want[0] == "ok" and isinstance(rd, Events):
        check_mark(rd, a, start, want[1]["mark"])
    return want


def check_mark(rd, a, start, mark):
    """the zxid high-water mark after reading `a`, on a context of its own (the mark outlives batches, so a shared
    context would compare against a running maximum)"""
    from registrar_b200 import _native
    c = _native.Context(0)
    try:
        c.register_batch(rd.batch)
        if rd.gate:
            assert c.setwatches_requests().relative_zxid == 0
        c.read_events(a, start=start, xid_base=rd.xb, n_xids=rd.nx)
        assert c.setwatches_requests().relative_zxid == mark, (rd.name, mark)
    finally:
        c.close()


# ------------------------------------------------------------------------------------------------------------ CPU --

@pytest.mark.parametrize("seed", range(4))
def test_generators_against_the_restatements(seed):
    paths, pays = cpu_paths(40)
    rng = random.Random(seed)
    for rd in readers(paths, pays, xb=[1, -2 ** 31, 2 ** 31 - 20][seed % 3]):
        # every unmutated stream is accepted
        for _ in range(3):
            b = honest_stream(rd, rng, trailing=False)
            assert rd.want(b)[0] == "ok", rd.name
            if rd.has_start:
                st = rng.randrange(64)
                assert rd.want(with_front(rd, b, st, rng), st)[0] == "ok", rd.name
        # a frame head at every phase of a span's last block
        for ph in range(16):
            b, at = span_phase_stream(rd, rng, 1, ph)
            assert at % fz.SPAN == fz.SPAN - 16 + ph and at in fz.cands(rd.head, b)
            assert rd.want(b)[0] == "ok"
        # stream lengths at span and super-tile multiples
        for L in (3 * fz.SPAN, fz.SUPER_BYTES):
            b = length_stream(rd, rng, L)
            assert len(b) == L and rd.want(b)[0] == "ok"


@pytest.mark.parametrize("n", [1, 6])
def test_every_candidate_count_is_built(n):
    """chain_to builds every listed C for every reader (it asserts the count with the reader's plausibility test):
    all on the chain (accepted, or refused where too few replies fit), and all but the chain false"""
    rng = random.Random(n)
    for rd in readers(*cpu_paths(n), xb=7):
        for C in [c for c in CS if (n == 1 or c >= 8) and c <= 1025] + [(1 << 17) + 1] * (n == 1):
            for false in (False, True):
                b = chain_to(rd, rng, C, false)
                if C > 4 and not false:
                    assert rd.want(b)[0] == "ok", (rd.name, C)


def test_children_reach_is_planted():
    """a one-record batch's only directory lists exactly `count` entries, the largest count of the stream"""
    rng = random.Random(2)
    for count in (1, 2, 3, 7, 8, 9, 4095):
        rd = Children(*cpu_paths(1), 1, count)
        for b in (honest_stream(rd, rng, noise=False, decoys=False, trailing=False), honest_stream(rd, rng, trailing=False)):
            w = rd.want(b)
            assert w[0] == "ok" and max(np.diff(w[1]["off"])) == count


def test_long_front_chains_past_start():
    rng = random.Random(1)
    for st in range(0, 300, 1):
        f = fz.long_front(st, rng)
        b = f + ru.ping() * 4
        assert len(f) == st
        if st < 8:
            assert not fz.cands(lambda b, p: ru.plausible(b, p, 1, 1), f + b"\xff" * 8)
            continue
        pos = 0
        while pos < st:          # the replies readers' test; from 32 bytes on the events reader's too
            assert ru.plausible(b, pos, 1, 1) == ru.OK
            if st >= 32:
                assert eu.head(b, pos, 0, 0) == eu.OK
            pos += 4 + fz.be32(b, pos)
        assert pos == max(st + 7, 20)


def span_phase_stream(rd, rng, s, ph):
    """honest replies with a notification padded so that reply 1's head sits at byte s * 2048 - 16 + ph"""
    fr = plain_frames(rd, rng)
    at = s * fz.SPAN - 16 + ph
    head = fr[0]
    pad = fz.pad_to(len(head), at)
    return head + pad + b"".join(fr[1:]), at


def length_stream(rd, rng, L):
    """honest replies, then a trailing notification that makes the stream exactly L bytes"""
    b = b"".join(plain_frames(rd, rng))
    assert L - len(b) >= 32
    return b + fz.pad_to(len(b), L)


# ------------------------------------------------------------------------------------------------------------ GPU --

@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def setup(ctx, name, n=40, xb=1, seed=3, big=0):
    """register a fleet batch, frame what `name` reads, check the framing against the restatement -> the reader"""
    from registrar_b200.batch import RecordBatch
    from test_reconcile import run
    b = RecordBatch.from_records(fleet(n, seed=seed))
    paths, pays = run(ctx, b)
    rd = next(r for r in readers(paths, pays, xb) if r.name == name)
    if big and isinstance(rd, Children):
        rd = Children(paths, pays, xb, big)
    rd.batch = b
    assert rd.frame_on(ctx) == rd.framing()
    return rd


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("seed", range(4))
def test_random_and_mutated_streams(ctx, name, seed):
    random_cases(ctx, name, seed)


def random_cases(ctx, name, seed, count=24):
    rng = random.Random(zlib.crc32(b"%s-%d" % (name.encode(), seed)))
    rd = setup(ctx, name, n=rng.choice([8, 40, 90]), seed=seed)
    for _ in range(count):
        b = honest_stream(rd, rng)
        start = 0
        if rd.has_start and rng.randrange(2):
            start = rng.choice([rng.randrange(16), rng.randrange(100), fz.SPAN])
            b = with_front(rd, b, start, rng)
        b, _ = fz.mutate(b, rng, 3, start)
        run_case(ctx, rd, b, start)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_frame_heads_across_span_boundaries(ctx, name):
    rng = random.Random(5)
    rd = setup(ctx, name)
    for s in (1, 2, 64):
        for ph in range(16):
            b, at = span_phase_stream(rd, rng, s, ph)
            run_case(ctx, rd, b)
            run_case(ctx, rd, b[:at + rng.randrange(1, 24)])          # cut just past the head: refused or partial


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_stream_lengths(ctx, name):
    rng = random.Random(6)
    rd = setup(ctx, name, n=12)
    b = honest_stream(rd, rng, noise=False, decoys=False, trailing=False)
    for L in range(25):
        run_case(ctx, rd, b[:L])
        run_case(ctx, rd, ru.ping()[:L])
    for L in (fz.SPAN, 2 * fz.SPAN, fz.SUPER_BYTES, 2 * fz.SUPER_BYTES):
        s = length_stream(rd, rng, L)
        for cut in (-1, 0):
            run_case(ctx, rd, s[:L + cut])
        run_case(ctx, rd, s + b"\0")


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_candidate_counts(ctx, name):
    rng = random.Random(7)
    rd = setup(ctx, name, n=1)
    for C in CS:
        for false in (False, True):
            run_case(ctx, rd, chain_to(rd, rng, C, false))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("name", NAMES)
def test_candidate_counts_large(ctx, name):
    rng = random.Random(8)
    rd = setup(ctx, name, n=6)
    for m in range(18, 21):
        for C in (2 ** m - 1, 2 ** m, 2 ** m + 1):
            for false in (False, True):
                run_case(ctx, rd, chain_to(rd, rng, C, false))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("seed", range(4, 24))
def test_random_and_mutated_streams_sweep(ctx, name, seed):
    random_cases(ctx, name, seed, count=48)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in NAMES if n != "replies"])
def test_start_phases(ctx, name):
    rng = random.Random(9)
    rd = setup(ctx, name, n=20)
    b = honest_stream(rd, rng, trailing=False)
    for start in list(range(16)) + [16 * rng.randrange(2, 40) + ph for ph in range(16)] + [fz.SPAN, fz.SPAN + 1, 2 * fz.SPAN]:
        s = with_front(rd, b, start, rng)
        run_case(ctx, rd, s, start)
        run_case(ctx, rd, s[:start + 9], start)
    run_case(ctx, rd, b + b"", len(b))          # start at the end: nothing to read


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_device_view_inside_a_larger_buffer(ctx, name):
    """the bytes past the view complete the last frame: a reader that used them would accept what the restatement
    refuses (or, for events, read a frame the restatement calls partial)"""
    rng = random.Random(10)
    rd = setup(ctx, name, n=20)
    for _ in range(6):
        fr = rd.frames(rng)             # the last frame: the reply to the last record (events: a notification)
        last = fr[-1]
        b = b"".join(fz.interleave(fr[:-1], rng, fz.noise(rng, rd.paths, 4))) + last
        cuts = {1, 2, 3, 4, 5, 8, 15, 16, 17, 19, 20, rng.randrange(1, len(last))} | {len(last) - k for k in (0, 1, 4, 5, 16, 20)}
        for cut in sorted(c for c in cuts if 1 <= c <= len(last)):
            run_case(ctx, rd, b[:-cut], view=b[-cut:] + ru.ping())


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_xid_bases(ctx, name):
    from registrar_b200 import _native
    rng = random.Random(11)
    for xb in (-2 ** 31, 0, 2 ** 31 - 1, 2 ** 31 - 5, -2 ** 31 + 3):
        rd = setup(ctx, name, n=12, xb=xb)
        for _ in range(4):
            run_case(ctx, rd, fz.mutate(honest_stream(rd, rng), rng, 1)[0])
    if name.startswith("events"):
        rd = setup(ctx, name, n=12, xb=5)
        rd.nx = 0
        run_case(ctx, rd, honest_stream(rd, rng))
        run_case(ctx, rd, cu.error(5, 0) + ru.ping())
        for xb, nx in ((-3, 3), (-1, 1), (-2, 1), (2 ** 31 - 1, 2 ** 31)):
            rd.prepare(ctx)
            with pytest.raises(_native.RegkError) as e:
                ctx.read_events(np.frombuffer(ru.ping(), np.uint8), xid_base=xb, n_xids=nx)
            assert "which ZooKeeper uses for" in e.value.message
        return
    k = len(fz.split(setup(ctx, name, n=12).framing()))
    for xb in (-1, -2, -k):         # a framed range holding -1 or -2 is refused by the reader
        rd = setup(ctx, name, n=12, xb=xb)
        with pytest.raises(_native.RegkError) as e:
            rd.call(ctx, np.frombuffer(rd.honest(rng), np.uint8), 0, False)
        assert "which ZooKeeper uses for" in e.value.message


@pytest.mark.gpu
@pytest.mark.parametrize("gate", [False, True])
def test_events_in_chunks(ctx, gate):
    """one call and random chunks (each carrying the bytes from `consumed`) give the same events, counts and pending
    sets"""
    rng = random.Random(12)
    rd = setup(ctx, "events-gate" if gate else "events", n=40)
    for _ in range(6):
        b = honest_stream(rd, rng, trailing=False)
        want = rd.want(b)
        assert want[0] == "ok"
        rd.prepare(ctx)
        carry, fed, tot = b"", 0, [0, 0, 0]
        pos = []
        while fed < len(b):
            k = min(len(b), fed + rng.choice([1, 7, 20, 33, 100, 2048, 5000]))
            piece = carry + b[fed:k]
            base = fed - len(carry)
            g = ctx.read_events(np.frombuffer(piece, np.uint8), xid_base=rd.xb, n_xids=rd.nx)
            pos += [base + int(p) for p in g.pos]
            tot = [tot[0] + g.n_events, tot[1] + g.n_pings, tot[2] + g.n_replies]
            carry = piece[g.consumed:]
            fed = k
        assert not carry
        w = want[1]
        assert pos == w["pos"] and tot == w["counts"][:3]
        if not gate:
            assert pending(ctx) == w["pending"]


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 2, 3, 5, 8, 10, 12])
def test_children_listing_reach_at_powers_of_two(ctx, m):
    """a one-record batch whose only directory lists 2^m - 2, 2^m - 1 and 2^m entries: the entry chain's reach (the
    longest count + 1) at and beside a power of two"""
    rng = random.Random(13)
    for count in (2 ** m - 2, 2 ** m - 1, 2 ** m):
        if count < 1:
            continue
        rd = setup(ctx, "children", n=1, big=count)
        for b in (honest_stream(rd, rng, noise=False, decoys=False, trailing=False), honest_stream(rd, rng)):
            w = run_case(ctx, rd, b)
            assert w[0] == "ok" and max(np.diff(w[1]["off"])) == count
