"""Independent restatement of the watched heartbeat across a reconnect (regk_setwatches_requests and the SetWatches
replies regk_read_events accepts after it), for the tests: the SetWatches frames and their closed-form split, the watch
kinds and the re-pend rule, the session's zxid high-water mark with the reader's -8 test, and a ZooKeeper model with
per-connection watches that serves SetWatches as ZooKeeper 3.4's DataTree.setWatches does.  The layouts follow
zookeeper.jute (RequestHeader, SetWatches, ReplyHeader; integers big endian).  PARITY UNPINNED: pinned against a frame
and a reply worked out by hand, not against a server."""
import struct

import children_util as cu
import events_util as eu
import reconcile_owned_util as ou

SW_XID, SW_OP = -8, 101
DEFAULT_MAX_FRAME = 131072
OVERHEAD = 32
NONE, DATA, EXIST, CHILD = 0, 1, 2, 3
NONODE = ou.NONODE
SW_BODY, SW_ERR = eu.PING_BODY + 1, eu.PING_BODY + 2          # the reader's refusals beyond events_util's


def split(D, E, C, max_frame, lmax):
    """-> [[D_f, E_f, C_f] per frame]: entry j of D ++ E ++ C (4 + P bytes) goes into frame s_j // B"""
    L = 4 + lmax
    if max_frame == 0:
        max_frame = DEFAULT_MAX_FRAME
    assert max_frame >= OVERHEAD + 2 * L
    B = max_frame - OVERHEAD - L
    out, s = [], 0
    for lst, paths in enumerate((D, E, C)):
        for p in paths:
            f = s // B
            while len(out) <= f:
                out.append([[], [], []])
            out[f][lst].append(p)
            s += 4 + len(p)
    return out


def frames(D, E, C, rel_zxid, max_frame, lmax):
    """the SetWatches frames -> (bytes, offsets)"""
    out, off = b"", [0]
    for fr in split(D, E, C, max_frame, lmax):
        body = struct.pack(">iiq", SW_XID, SW_OP, rel_zxid)
        for lst in fr:
            body += struct.pack(">i", len(lst)) + b"".join(struct.pack(">i", len(p)) + p for p in lst)
        out += struct.pack(">i", len(body)) + body
        off.append(len(out))
    return out, off


def parse(frame_bytes):
    """SetWatches frames -> [(relativeZxid, D, E, C)]"""
    b, k, out = bytes(frame_bytes), 0, []
    while k < len(b):
        ln, xid, op, rel = struct.unpack_from(">iiiq", b, k)
        assert xid == SW_XID and op == SW_OP
        end, q, lists = k + 4 + ln, k + 20, []
        for _ in range(3):
            (cnt,) = struct.unpack_from(">i", b, q)
            q += 4
            lst = []
            for _ in range(cnt):
                (pl,) = struct.unpack_from(">i", b, q)
                lst.append(b[q + 4:q + 4 + pl])
                q += 4 + pl
            lists.append(lst)
        assert q == end
        out.append((rel, *lists))
        k = end
    return out


def reply(zxid, err=0, body=b""):
    """the SetWatches reply: a bare ReplyHeader (len 16) unless body is given"""
    h = struct.pack(">iqi", SW_XID, zxid, err) + body
    return struct.pack(">i", len(h)) + h


def stat_kind(err):
    """the kind an exists reply arms"""
    return DATA if err == 0 else EXIST if err == NONODE else NONE


def child_kind(err):
    """the kind a getChildren reply arms"""
    return CHILD if err == 0 else NONE


def lists(paths, rec_kind, dir_kind, pend_recs=(), pend_dirs=()):
    """rec_kind {record: kind}, dir_kind {directory k: kind} (missing = NONE: never armed, or in flight) ->
    (D, E, C as paths, re-pended records, re-pended directories): every first-of-path record and every directory of
    children_util.dir_set is listed by its kind or, when it is neither listed nor pending, re-pended"""
    first = {}
    for i, p in enumerate(paths):
        first.setdefault(p, i)
    dirs = [d for _, d in cu.dir_set(paths)[0]]
    D, E, rr = [], [], []
    for i in sorted(first.values()):
        if i in pend_recs:
            continue
        k = rec_kind.get(i, NONE)
        (D if k == DATA else E if k == EXIST else rr).append(paths[i] if k in (DATA, EXIST) else i)
    C, rd = [], []
    for k, d in enumerate(dirs):
        if k in pend_dirs:
            continue
        if dir_kind.get(k, NONE) == CHILD:
            C.append(d)
        else:
            rd.append(k)
    return D, E, C, rr, rd


def head(b, pos, xid_base, n_xids, gate):
    """regk_read_events' test of the frame at pos, with SetWatches replies accepted when the gate is open"""
    c = eu.head(b, pos, xid_base, n_xids)
    if not gate or c in (eu.TRUNC, eu.BAD_LEN) or eu._i32(b, pos + 4) != SW_XID:
        return c
    ln, err = eu._i32(b, pos), eu._i32(b, pos + 16)
    return SW_BODY if ln != 16 else SW_ERR if err else eu.OK


def read(stream, xid_base=0, n_xids=0, start=0, gate=False, mark=0):
    """the sequential reader -> dict(n_replies, n_pings, n_events, consumed, partial, mark): mark = max(mark, the
    ReplyHeader.zxid of every complete reply and SetWatches reply); raises eu.Refused (nothing is taken then)"""
    b = bytes(stream)
    pos, replies, pings, events, m = start, 0, 0, 0, mark
    while pos < len(b):
        c = head(b, pos, xid_base, n_xids, gate)
        if c == eu.TRUNC:
            return dict(n_replies=replies, n_pings=pings, n_events=events, consumed=pos, partial=True, mark=m)
        if c != eu.OK:
            raise eu.Refused(c, pos)
        xid = eu._i32(b, pos + 4)
        if xid == eu.NOTIFY_XID:
            events += 1
        elif xid == eu.PING_XID:
            pings += 1
        else:
            replies += 1
            m = max(m, struct.unpack_from(">q", b, pos + 8)[0])
        pos += 4 + eu._i32(b, pos)
    return dict(n_replies=replies, n_pings=pings, n_events=events, consumed=pos, partial=False, mark=m)


class SessionZooKeeper(eu.WatchedZooKeeper):
    """eu.WatchedZooKeeper whose nodes carry an mzxid (and directories a pzxid), whose reply headers carry the current
    zxid, whose watches die with the connection, and which serves SetWatches"""

    def __init__(self):
        super().__init__()
        self.mzxid, self.pzxid = {}, {}

    def _fire(self, ops):
        for op, path in ops:
            super()._fire([(op, path)])
            if op == ou.OP_CREATE:
                self.mzxid[path] = self.zxid
                self.pzxid[ou.parent(path)] = self.zxid
            elif op == ou.OP_DELETE:
                self.mzxid.pop(path, None)
                self.pzxid[ou.parent(path)] = self.zxid
            else:
                self.mzxid[path] = self.zxid

    def serve_reads(self, frame_bytes, session):
        b = bytearray(super().serve_reads(frame_bytes, session))
        k = 0
        while k < len(b):
            b[k + 8:k + 16] = struct.pack(">q", self.zxid)
            k += 4 + struct.unpack_from(">i", b, k)[0]
        return bytes(b)

    def drop_connection(self, session):
        """the connection's watches, and whatever it had not delivered yet, are gone"""
        self.data_w[session], self.child_w[session], self.queue[session] = set(), set(), []

    def serve_setwatches(self, frame_bytes, session):
        """DataTree.setWatches per frame: the events it fires, then its reply"""
        out = []
        for rel, D, E, C in parse(frame_bytes):
            for p in D:
                if p not in self.nodes:
                    out.append(eu.notification(p, eu.DELETED))
                elif self.mzxid.get(p, 0) > rel:
                    out.append(eu.notification(p, eu.DATA_CHANGED))
                else:
                    self.data_w.setdefault(session, set()).add(p)
            for p in E:
                if p in self.nodes:
                    out.append(eu.notification(p, eu.CREATED))
                else:
                    self.data_w.setdefault(session, set()).add(p)
            for p in C:
                if p not in self.nodes:
                    out.append(eu.notification(p, eu.DELETED))
                elif self.pzxid.get(p, 0) > rel:
                    out.append(eu.notification(p, eu.CHILDREN_CHANGED))
                else:
                    self.child_w.setdefault(session, set()).add(p)
            out.append(reply(self.zxid))
        return b"".join(out)
