"""Independent restatement of a watched walk carried across a reconnect (regk_walk_setwatches, the ARMED bit, the walk's
zxid high-water mark and the SetWatches gate of regk_walk_events), for the tests: a tree server that is
walk_watch_util.WalkZooKeeper and setwatches_util.SessionZooKeeper at once (mzxid / pzxid per node, the current zxid in
every reply header, watches and undelivered bytes lost on drop_connection, SetWatches served as DataTree.setWatches), a
sequential model of the walk state as include/regk.h states it, and a driver that drops the connection at chosen points,
mutates the tree while it is down and resumes.  PARITY UNPINNED: the server's rules as the two utilities restate them,
not a server."""
import struct

import children_util as cu
import events_util as ev
import replies_util as ru
import setwatches_util as sw
import walk_watch_util as ww

PENDING, REMOVED, NO_NODE = ww.PENDING, ww.REMOVED, ww.NO_NODE


class Refused(Exception):
    """a call the library refuses before it changes anything (the state or an argument)"""


class TreeZooKeeper(ww.WalkZooKeeper, sw.SessionZooKeeper):
    """the walk's tree server with sessions: every reply header carries the zxid current when it was sent, and
    fail[(op, path)] = err answers that read with an error (arming nothing)"""

    def __init__(self):
        super().__init__()
        self.fail = {}

    def serve(self, frame_bytes, session, during=None):
        out = [self.take_events(session)]
        for k, (xid, op, path, watch) in enumerate(ev.parse_reads(frame_bytes)):
            node, err = self.nodes.get(path), self.fail.get((op, path))
            if node is None or err is not None:
                r = ru.error(xid, ru.NONODE if node is None else err)
            elif op == ww.OP_GETDATA:
                if watch:
                    self.data_w.setdefault(session, set()).add(path)
                r = ru.success(xid, node.data, node.version, node.owner, len(self.kids[path]), seed=k)
            else:
                if watch:
                    self.child_w.setdefault(session, set()).add(path)
                r = cu.success(xid, list(self.kids[path]))
            out.append(r[:8] + struct.pack(">q", self.zxid) + r[16:])
            if during:
                during(k)
            out.append(self.take_events(session))
        return b"".join(out)


def frames_of(stream, start=0):
    """the complete frames of a stream from `start` -> [(pos, len, xid, zxid)]"""
    b, pos, out = bytes(stream), start, []
    while pos + 4 <= len(b):
        (ln,) = struct.unpack_from(">i", b, pos)
        if ln < 16 or pos + 4 + ln > len(b):
            break
        xid, zxid = struct.unpack_from(">iq", b, pos + 4)
        out.append((pos, ln, xid, zxid))
        pos += 4 + ln
    return out


def read_events(stream, xid_base, n_xids, start, gate):
    """regk_walk_events' frame reader with the gate: ev.read, with a SetWatches reply (xid -8, len 16, err 0) accepted
    as a reply while the gate is open -> ev.read's dict plus `mark` (the largest reply zxid); raises ev.Refused"""
    b = bytes(stream)
    pos, events, pings, replies, mark = start, [], 0, 0, 0
    while pos < len(b):
        c = sw.head(b, pos, xid_base, n_xids, gate)
        if c == ev.TRUNC:
            return dict(events=events, n_pings=pings, n_replies=replies, consumed=pos, partial=True, mark=mark)
        if c != ev.OK:
            raise ev.Refused(c, pos)
        ln, xid = struct.unpack_from(">ii", b, pos)
        if xid == ev.NOTIFY_XID:
            typ, state, plen = struct.unpack_from(">iii", b, pos + 20)
            events.append((pos, typ, state, struct.unpack_from(">q", b, pos + 8)[0], b[pos + 32:pos + 32 + plen]))
        elif xid == ev.PING_XID:
            pings += 1
        else:
            replies += 1
            mark = max(mark, struct.unpack_from(">q", b, pos + 8)[0])
        pos += 4 + ln
    return dict(events=events, n_pings=pings, n_replies=replies, consumed=pos, partial=False, mark=mark)


class Model(ww.Model):
    """ww.Model with the ARMED bit per node, the walk's zxid mark and the SetWatches gate"""

    def start(self, roots):
        super().start(roots)
        self.armed, self.mark, self.gate = [], 0, False

    def _drop_removed(self, replaced=None):
        keep = [j for j in range(len(self.nodes)) if not self.marks[j] & REMOVED]
        self.armed = [self.armed[j] for j in keep]
        super()._drop_removed(replaced)

    def read(self, stream):
        f, xb = len(self.frontier), self.xid
        r1 = ru.read(stream, xb, f)
        r2 = cu.read(stream, ww.wrap(xb + f), f, start=r1["consumed"])
        w = self.framed_watch
        if self.fnode is not None:                      # a refresh level: through fnode, before the rebuild
            for i, j in enumerate(self.fnode):
                self.armed[j] = w and r1["err"][i] == 0 and r2["err"][i] == 0
            want = super().read(stream)
        else:
            want = super().read(stream)
            self.armed += [w and r2["err"][k] == 0 for k, _, _, _ in r1["found"]]
        zx = [z for _, _, xid, z in frames_of(stream) if xid not in (ev.NOTIFY_XID, ev.PING_XID)]
        self.mark = max([self.mark] + zx)
        return want

    def events(self, stream, start=0, xid_base=0, n_xids=0):
        """regk_walk_events with the gate; raises ev.Refused"""
        r = read_events(stream, xid_base, n_xids, start, self.gate)
        present = {self.nodes[j][0]: j for j in range(len(self.nodes)) if not self.marks[j] & REMOVED}
        out, unmatched, other, pend, gone = [], 0, 0, [], []
        for pos, typ, state, zxid, path in r["events"]:
            j = present.get(path) if typ in (ev.DELETED, ev.DATA_CHANGED, ev.CHILDREN_CHANGED) else None
            if j is None:
                unmatched += 1
            elif typ == ev.DELETED:
                gone.append(j)
                d = path[:max(path.rfind(b"/"), 0)]
                if d and d in present:
                    pend.append(present[d])
            else:
                pend.append(j)
            other += typ == ev.NONE or typ >= 5
            out.append((pos, typ, state, zxid, NO_NODE if j is None else j))
        for j in pend:
            self.marks[j] |= PENDING
        for j in gone:
            self.marks[j] |= REMOVED
        self.mark = max(self.mark, r["mark"])
        n_pending, n_removed = self.counts()
        return dict(events=out, n_events=len(out), n_pings=r["n_pings"], n_replies=r["n_replies"], n_unmatched=unmatched,
                    n_other=other, consumed=r["consumed"], partial=r["partial"], n_pending=n_pending, n_removed=n_removed)

    def lmax(self):
        return max((len(n[0]) for n in self.nodes), default=0)

    def setwatches(self, max_frame=0, frames=True):
        """regk_walk_setwatches -> dict(n_listed, n_repend, n_pending, n_removed, n_frontier, relative_zxid, frames,
        frame_off, listed); raises Refused as the library refuses (changing nothing).  frames=False leaves the frames
        out (None), for very large snapshots"""
        if not self.watched:
            raise Refused("unwatched")
        mf = max_frame or sw.DEFAULT_MAX_FRAME
        if mf >= 2 ** 31 or mf < sw.OVERHEAD + 2 * (4 + self.lmax()):
            raise Refused("max_frame")
        front = set(self.fnode or ())
        listed, repend = [], []
        for j in range(len(self.nodes)):
            if self.marks[j] or j in front:
                continue
            (listed if self.armed[j] else repend).append(j)
        for j in repend:
            self.marks[j] |= PENDING
        D = [self.nodes[j][0] for j in listed]
        fb, off = sw.frames(D, [], D, self.mark, max_frame, self.lmax()) if frames else (None, None)
        self.gate = True
        n_pending, n_removed = self.counts()
        return dict(n_listed=len(listed), n_repend=len(repend), n_pending=n_pending, n_removed=n_removed,
                    n_frontier=len(self.frontier), relative_zxid=self.mark, frames=fb, frame_off=off, listed=listed)


MODES = ("between", "tail", "refresh_unread", "pending")


class Driver(ww.Driver):
    """ww.Driver over a TreeZooKeeper and this Model; lib (optional) also gets lib.setwatches(max_frame, want)"""

    def __init__(self, zk, roots, rng, lib=None):
        super().__init__(zk, roots, rng, lib)
        self.model = Model()

    def setwatches(self, max_frame=0):
        want = self.model.setwatches(max_frame)
        if self.lib:
            self.lib.setwatches(max_frame, want)
        return want

    def cut_level(self, deliver):
        """frame the current frontier and let the server answer it, but lose the connection with only a prefix of the
        reply bytes delivered (fed with the level's reply range when `deliver`, else discarded)"""
        f = len(self.model.frontier)
        xb = self._next_xid(2 * f)
        frames = self.model.requests(xb, True)
        if self.lib:
            self.lib.requests(xb, True, frames)
        stream = self.zk.serve(frames, self.SESSION)
        cut = self.rng.randrange(len(stream) + 1)
        if deliver and cut:
            self._events(stream[:cut], 0, xb, 2 * f)

    def refresh_framed(self):
        """walk_refresh, leaving the refresh level unframed"""
        want = self.model.refresh()
        if self.lib:
            self.lib.refresh(want, self.model)
        return want

    def drop(self, mode, mut, churn):
        """lose the connection at the point `mode` names (between levels; with the tail of a level's replies lost;
        with a refresh level framed but unread; with pending nodes not yet refreshed), then mutate the tree while it is
        down"""
        rng = self.rng
        if mode == "tail" and self.model.frontier:
            self.cut_level(rng.random() < 0.5)
        elif mode in ("refresh_unread", "pending") and not self.model.frontier:
            mut.some(1 + rng.randrange(churn + 1))
            self.feed(self.zk.take_events(self.SESSION))
            if mode == "refresh_unread" and self.model.counts() != (0, 0):
                self.refresh_framed()
                if self.model.frontier and rng.random() < 0.8:
                    self.cut_level(rng.random() < 0.5)
        self.zk.drop_connection(self.SESSION)
        mut.some(churn)


def script(rng, lib=None, drops=3, depth=3, fan=(0, 1, 2, 4), churn=4, roots=(b"/z",), max_frame=0):
    """a random script of walks, refreshes and connection drops to convergence -> the Driver; asserts that after every
    resume the pending and removed nodes are exactly those the drop left pending or removed, those re-pended, and the
    listed nodes that changed while the connection was down, and that the settled snapshot equals the tree"""
    zk = TreeZooKeeper()
    for r in roots:
        ww.build_tree(zk, rng, r, depth, fan)
    d = Driver(zk, roots, rng, lib)
    mut = ww.Mutator(zk, roots, rng)
    d.model.start(d.roots)
    if lib:
        lib.start(d.roots)
    for _ in range(drops):
        for _ in range(rng.randrange(4)):                 # some of the way: whole levels, sometimes a refresh round
            if d.model.frontier:
                d.level()
        if not d.model.frontier and rng.random() < 0.4:
            mut.some(rng.randrange(churn + 1))
            d.feed(zk.take_events(d.SESSION))
            d.refresh(mut.in_flight(0.05))
        d.drop(rng.choice(MODES), mut, rng.randrange(churn + 1))
        check_resume(d, max_frame)
    d.levels()
    d.settle()
    assert d.snapshot_set() == zk.subtree(roots)
    return d


def changed_while_down(zk, path, rel):
    return path not in zk.nodes or zk.mzxid.get(path, 0) > rel or zk.pzxid.get(path, 0) > rel


def check_resume(d, max_frame=0):
    """resume and check the pending-and-removed set it leaves"""
    m = d.model
    before = {j for j in range(len(m.nodes)) if m.marks[j]}
    want = d.setwatches(max_frame)
    rel = want["relative_zxid"]
    moved = {j for j in want["listed"] if changed_while_down(d.zk, m.nodes[j][0], rel)}
    present = {m.nodes[j][0]: j for j in range(len(m.nodes)) if not m.marks[j] & REMOVED}
    for j in want["listed"]:                             # NodeDeleted makes the parent pending
        p = m.nodes[j][0]
        if p not in d.zk.nodes and p[:p.rfind(b"/")] in present:
            moved.add(present[p[:p.rfind(b"/")]])
    repend = {j for j in range(len(m.nodes)) if m.marks[j] and j not in before}
    stream = d.zk.serve_setwatches(want["frames"], d.SESSION)
    d.feed(stream)
    assert sum(1 for f in frames_of(stream) if f[2] == sw.SW_XID) == len(want["frame_off"]) - 1
    after = {j for j in range(len(m.nodes)) if m.marks[j]}
    assert after == before | repend | moved, (sorted(after), sorted(before | repend | moved))
    d.levels()
    return want


PATHS_README = [b"/us/joyent", b"/us/joyent/emy-10", b"/us/joyent/emy-10/authcache"]


def readme_walked(lib=None, rng=None):
    """the README's authcache tree walked from /us/joyent with watches -> (zk, Driver)"""
    import random

    import walk_util as wu
    zk = TreeZooKeeper()
    t = wu.readme_tree()
    for p in sorted(t.nodes, key=len):
        zk.create(p, t.nodes[p][0], 0, False)
    d = Driver(zk, [b"/us/joyent"], rng or random.Random(0), lib)
    d.start()
    return zk, d


def struct_fields(header, name):
    """the field names of `typedef struct name { ... } name;` in include/regk.h, in order"""
    body = header.split("typedef struct %s {" % name)[1].split("} %s;" % name)[0]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip().rstrip(";")
        if line:
            fields += [f.strip().lstrip("*").strip() for f in line.split(None, 1)[1].split(",")]
    return fields
