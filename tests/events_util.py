"""Independent restatement of the watched heartbeat (REGK_ZK_WATCH, regk_read_events, regk_events_requests), for the
tests: read frames with their watch byte, the notification builder, a sequential reader of a session stream with the
refusal codes, the mapping of events to records and service directories with the pending sets, and a watch-aware
ZooKeeper model built over reconcile_owned_util.ZooKeeper.  The layouts follow zookeeper.jute (ReplyHeader,
WatcherEvent, ExistsRequest, GetDataRequest, GetChildrenRequest; integers big endian) and the server's watch rules:
watches are one-shot and per session; a create fires NodeCreated on the node and NodeChildrenChanged on its parent, a
delete NodeDeleted on the node (its data and child watches alike, once) and NodeChildrenChanged on its parent, a
setData NodeDataChanged; a multi fires per operation, and only when it commits.  PARITY UNPINNED: pinned against
operations worked out by hand, not against a server."""
import struct

import children_util as cu
import reconcile_owned_util as ou
import replies_util as ru
import stats_util as su

NOTIFY_XID, PING_XID = -1, -2
NONE, CREATED, DELETED, DATA_CHANGED, CHILDREN_CHANGED = -1, 1, 2, 3, 4
SYNC_CONNECTED = 3
SUBJ_NONE, SUBJ_RECORD, SUBJ_DIR = 0, 1, 2
NO_SUBJECT = 2 ** 64 - 1

# refusal codes, as regk_events.cuh numbers them
OK, TRUNC, BAD_LEN, NEG_XID, XID_RANGE, NOTE_LEN, NEG_PATH, NOTE_ERR, TYPE, PING_BODY = range(10)

wrap, ping = ru.wrap, ru.ping


def read_frames(op, paths, xid_base=1, watch=False):
    """len | RequestHeader{xid_base + i, op} | {path i, watch}: ExistsRequest (3), GetDataRequest (4), GetChildrenRequest (8)"""
    out = []
    for i, p in enumerate(paths):
        body = struct.pack(">ii", wrap(xid_base + i), op) + struct.pack(">i", len(p)) + p + (b"\x01" if watch else b"\x00")
        out.append(struct.pack(">i", len(body)) + body)
    return b"".join(out)


def parse_reads(frame_bytes):
    """read frames -> [(xid, op, path, watch)]"""
    b, k, out = bytes(frame_bytes), 0, []
    while k < len(b):
        ln, xid, op, pl = struct.unpack_from(">iiii", b, k)
        assert op in (3, 4, 8) and ln == 13 + pl and b[k + 16 + pl] in (0, 1)
        out.append((xid, op, b[k + 16:k + 16 + pl], b[k + 16 + pl]))
        k += 4 + ln
    return out


def notification(path, typ=DATA_CHANGED, state=SYNC_CONNECTED, zxid=-1, err=0, plen=None):
    """len | ReplyHeader{-1, zxid, err} | WatcherEvent{type, state, path}; plen overrides the path's length word"""
    body = struct.pack(">iqi", NOTIFY_XID, zxid, err)
    body += struct.pack(">iii", typ, state, len(path) if plen is None else plen) + path
    return struct.pack(">i", len(body)) + body


class Refused(Exception):
    def __init__(self, code, pos):
        super().__init__("code %d at byte %d" % (code, pos))
        self.code, self.pos = code, pos


def _i32(b, k):
    return struct.unpack_from(">i", b, k)[0]


def head(b, pos, xid_base, n_xids):
    """the test regk_read_events applies to the frame at `pos` -> OK or a code (TRUNC: the frame is still arriving)"""
    avail = len(b) - pos
    if avail < 4:
        return TRUNC
    ln = _i32(b, pos)
    if ln < 16:
        return BAD_LEN
    if ln + 4 > avail:
        return TRUNC
    xid, err = _i32(b, pos + 4), _i32(b, pos + 16)
    if xid == PING_XID:
        return OK if ln == 16 else PING_BODY
    if xid == NOTIFY_XID:
        if ln < 28:
            return NOTE_LEN
        typ, plen = _i32(b, pos + 20), _i32(b, pos + 28)
        if plen < 0:
            return NEG_PATH
        if plen != ln - 28:
            return NOTE_LEN
        if err != 0:
            return NOTE_ERR
        return OK if -1 <= typ <= 7 else TYPE
    if (xid - xid_base) % 2 ** 32 < n_xids:
        return OK
    return NEG_XID if xid < 0 else XID_RANGE


def read(stream, xid_base=0, n_xids=0, start=0):
    """the sequential reader: -> dict(events [(pos, type, state, zxid, path)], n_pings, n_replies, consumed, partial);
    raises Refused at the first frame that fails"""
    b = bytes(stream)
    pos, events, pings, replies = start, [], 0, 0
    while pos < len(b):
        c = head(b, pos, xid_base, n_xids)
        if c == TRUNC:
            return dict(events=events, n_pings=pings, n_replies=replies, consumed=pos, partial=True)
        if c != OK:
            raise Refused(c, pos)
        ln, xid = _i32(b, pos), _i32(b, pos + 4)
        if xid == NOTIFY_XID:
            typ, state, plen = struct.unpack_from(">iii", b, pos + 20)
            events.append((pos, typ, state, struct.unpack_from(">q", b, pos + 8)[0], b[pos + 32:pos + 32 + plen]))
        elif xid == PING_XID:
            pings += 1
        else:
            replies += 1
        pos += 4 + ln
    return dict(events=events, n_pings=pings, n_replies=replies, consumed=pos, partial=False)


class Mapper:
    """the subjects and pending sets of one batch generation: record table = first record per path, directory k = the
    k-th listed directory of children_util.dir_set"""

    def __init__(self, paths):
        self.first = {}
        for i, p in enumerate(paths):
            self.first.setdefault(p, i)
        self.dirs = {d: k for k, (_, d) in enumerate(cu.dir_set(paths)[0])}
        self.dirty_recs, self.dirty_dirs = {}, set()

    def subject(self, typ, path):
        if typ in (CREATED, DELETED, DATA_CHANGED) and path in self.first:
            return SUBJ_RECORD, self.first[path]
        if typ in (DELETED, CHILDREN_CHANGED) and path in self.dirs:
            return SUBJ_DIR, self.dirs[path]
        return SUBJ_NONE, NO_SUBJECT

    def feed(self, events):
        """-> [(kind, subject)] per event, marking the subjects; plus (n_unmatched, n_other)"""
        out, unmatched, other = [], 0, 0
        for _, typ, _, _, path in events:
            kind, s = self.subject(typ, path)
            if kind == SUBJ_RECORD:
                self.dirty_recs[s] = self.dirty_recs.get(s, 0) | 1 << (typ - 1)
            elif kind == SUBJ_DIR:
                self.dirty_dirs.add(s)
            else:
                unmatched += 1
            other += typ == NONE or typ >= 5
            out.append((kind, s))
        return out, unmatched, other

    def take(self, dirs=False):
        """the pending records (or directories), ascending; the set is then empty"""
        if dirs:
            out, self.dirty_dirs = sorted(self.dirty_dirs), set()
        else:
            out, self.dirty_recs = sorted(self.dirty_recs), {}
        return out


class WatchedZooKeeper(ou.ZooKeeper):
    """ou.ZooKeeper with one-shot data (exists and getData) and child watches per session; every fired watch queues a
    notification for its session."""

    def __init__(self):
        super().__init__()
        self.data_w, self.child_w, self.queue = {}, {}, {}
        self.zxid = 0x100000000
        self._ops = None

    def _apply(self, nodes, op, path, data, arg, session):
        rc = super()._apply(nodes, op, path, data, arg, session)
        if rc == ou.ZOK and self._ops is not None:
            self._ops.append((op, path))
        return rc

    def _fire(self, ops):
        for op, path in ops:
            self.zxid += 1
            if op == ou.OP_CREATE:
                self._trigger(self.data_w, path, CREATED)
                self._trigger(self.child_w, ou.parent(path), CHILDREN_CHANGED)
            elif op == ou.OP_DELETE:
                got = self._trigger(self.data_w, path, DELETED)
                self._trigger(self.child_w, path, DELETED, skip=got)
                self._trigger(self.child_w, ou.parent(path), CHILDREN_CHANGED)
            else:
                self._trigger(self.data_w, path, DATA_CHANGED)

    def _trigger(self, table, path, typ, skip=()):
        fired = set()
        for s, paths in table.items():
            if path in paths:
                paths.discard(path)
                fired.add(s)
                if s not in skip:
                    self.queue.setdefault(s, []).append(notification(path, typ, zxid=self.zxid))
        return fired

    def _run(self, fn):
        self._ops = []
        rc = fn()
        ops, self._ops = self._ops, None
        if rc == ou.ZOK:
            self._fire(ops)
        return rc

    def create(self, path, data, session, ephemeral=True):
        return self._run(lambda: super(WatchedZooKeeper, self).create(path, data, session, ephemeral))

    def delete(self, path, version=-1):
        return self._run(lambda: super(WatchedZooKeeper, self).delete(path, version))

    def set_data(self, path, data, version=-1):
        return self._run(lambda: super(WatchedZooKeeper, self).set_data(path, data, version))

    def apply_frame(self, frame, session):
        return self._run(lambda: super(WatchedZooKeeper, self).apply_frame(frame, session))

    def serve_reads(self, frame_bytes, session):
        """answer exists / getChildren read frames and arm the watches their watch byte asks for -> reply bytes"""
        out = []
        for xid, op, path, watch in parse_reads(frame_bytes):
            node = self.nodes.get(path)
            if op == 3:
                if watch:
                    self.data_w.setdefault(session, set()).add(path)          # an exists watch arms a missing node too
                if node is None:
                    out.append(ru.error(xid, ou.NONODE))
                else:
                    kids = sum(1 for p in self.nodes if ou.parent(p) == path)
                    out.append(su.success(xid, node.version, node.owner, len(node.data), kids, seed=su.node_seed(node)))
            elif op == 8:
                if node is None:
                    out.append(ru.error(xid, ou.NONODE))
                else:
                    if watch:
                        self.child_w.setdefault(session, set()).add(path)
                    out.append(cu.success(xid, cu.list_children(self, path)))
            else:
                raise ValueError("only exists and getChildren are served")
        return b"".join(out)

    def take_events(self, session):
        q, self.queue[session] = self.queue.get(session, []), []
        return b"".join(q)
