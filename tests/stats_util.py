"""Independent restatement of regk_jute_requests(REGK_ZK_EXISTS), regk_read_stats and regk_reconcile_stats, for the
tests: an ExistsRequest frame builder, a reply builder that answers parsed exists frames from the ZooKeeper model of
reconcile_owned_util, a sequential reader of the reply stream with the refusal codes, and the classification table.  The
layouts follow zookeeper.jute (RequestHeader, ExistsRequest, ReplyHeader, ExistsResponse, Stat; all integers big endian).
PARITY UNPINNED: they are pinned against frames worked out by hand from those definitions, not against a server."""
import struct
import zlib

import reconcile_owned_util as ou
import replies_util as ru

OP_EXISTS = 3
NOTIFY_XID, PING_XID = -1, -2
ZOK, NONODE = ou.ZOK, ou.NONODE
SAME, CREATE, UPDATE, DUP, REPLACE = ou.SAME, ou.CREATE, ou.UPDATE, ou.DUP, ou.REPLACE
NO_MATCH = 2 ** 64 - 1

# refusal codes, as regk_stats.cuh numbers them
OK, TRUNC, BAD_LEN, NEG_XID, XID_RANGE, ERR_BODY, SUCC_LEN, ORDER, NEG_DLEN = range(9)

wrap = ru.wrap
error, notification, ping = ru.error, ru.notification, ru.ping


def exists_frames(paths, xid_base=1):
    """len | RequestHeader{xid_base + i, 3} | ExistsRequest{path i, watch = false}, back to back"""
    out = []
    for i, p in enumerate(paths):
        body = struct.pack(">ii", wrap(xid_base + i), OP_EXISTS) + struct.pack(">i", len(p)) + p + b"\x00"
        out.append(struct.pack(">i", len(body)) + body)
    return b"".join(out)


def parse_exists(frame_bytes):
    """exists frames -> [(xid, path)]"""
    b, k, out = bytes(frame_bytes), 0, []
    while k < len(b):
        ln, xid, op, pl = struct.unpack_from(">iiii", b, k)
        assert op == OP_EXISTS and ln == 13 + pl and b[k + 16 + pl] == 0
        out.append((xid, b[k + 16:k + 16 + pl]))
        k += 4 + ln
    return out


def node_seed(node):
    """what a node's zxids are derived from: every write of the model changes its version or its data"""
    return (node.version & 0xFFFFFFFF) * 65536 + (zlib.crc32(node.data) & 0xFFFF)


def success(xid, version=0, owner=0, data_len=0, children=0, seed=0, zxid=None):
    """an ExistsResponse reply frame: ReplyHeader + the Stat of replies_util.stat"""
    body = struct.pack(">iqi", xid, 0x200000000 + (seed & 0xFFFF) if zxid is None else zxid, ZOK)
    body += ru.stat(version, owner, data_len, children, seed)
    return struct.pack(">i", len(body)) + body


def replies(zk, frame_bytes, errors=None, extra=None, trailing=b""):
    """answer every exists frame from the model `zk`: the node's Stat, or NONODE.  errors = {record: err} replaces
    record k's reply by an error reply; extra = {record: bytes} inserts frames before record k's reply (record n: after
    the last one); trailing is appended."""
    errors, extra = errors or {}, extra or {}
    out = []
    reqs = parse_exists(frame_bytes)
    for k, (xid, path) in enumerate(reqs):
        out.append(extra.get(k, b""))
        node = zk.nodes.get(path)
        if k in errors:
            out.append(error(xid, errors[k]))
        elif node is None:
            out.append(error(xid, NONODE))
        else:
            kids = sum(1 for p in zk.nodes if p.startswith(path + b"/") and b"/" not in p[len(path) + 1:])
            out.append(success(xid, node.version, node.owner, len(node.data), kids, seed=node_seed(node)))
    out.append(extra.get(len(reqs), b""))
    return b"".join(out) + trailing


class Refused(Exception):
    def __init__(self, code, pos, k):
        super().__init__("code %d at byte %d, record %d" % (code, pos, k))
        self.code, self.pos, self.k = code, pos, k


def _i32(b, k):
    return struct.unpack_from(">i", b, k)[0]


def _i64(b, k):
    return struct.unpack_from(">q", b, k)[0]


def plausible(b, pos, xid_base, n):
    """the plausibility test of regk_read_stats at `pos` -> OK or the refusal code"""
    avail = len(b) - pos
    if avail < 4:
        return TRUNC
    ln = _i32(b, pos)
    if ln < 16:
        return BAD_LEN
    if ln + 4 > avail:
        return TRUNC
    xid, err = _i32(b, pos + 4), _i32(b, pos + 16)
    if xid in (NOTIFY_XID, PING_XID):
        return OK
    if (xid - xid_base) % 2 ** 32 >= n:
        return NEG_XID if xid < 0 else XID_RANGE
    if err != 0:
        return OK if ln == 16 else ERR_BODY
    return OK if ln == 84 else SUCC_LEN


def read(stream, xid_base, n, start=0):
    """the sequential reader from `start`: -> dict(err, version, owner, data_length, mzxid, n_found, n_missing, n_error,
    n_skipped, consumed); raises Refused at the first frame that fails"""
    b = bytes(stream)
    pos, k, skipped = start, 0, 0
    err, ver, own, dlen, mz = [], [], [], [], []
    while k < n:
        c = plausible(b, pos, xid_base, n)
        if c != OK:
            raise Refused(c, pos, k)
        ln, xid, e = _i32(b, pos), _i32(b, pos + 4), _i32(b, pos + 16)
        if xid in (NOTIFY_XID, PING_XID):
            skipped += 1
            pos += 4 + ln
            continue
        if xid != wrap(xid_base + k):
            raise Refused(ORDER, pos, k)
        if e == 0:
            if _i32(b, pos + 72) < 0:
                raise Refused(NEG_DLEN, pos, k)
            ver.append(_i32(b, pos + 52))
            own.append(_i64(b, pos + 64))
            dlen.append(_i32(b, pos + 72))
            mz.append(_i64(b, pos + 28))
        else:
            ver.append(0), own.append(0), dlen.append(0), mz.append(0)
        err.append(e)
        k += 1
        pos += 4 + ln
    return dict(err=err, version=ver, owner=own, data_length=dlen, mzxid=mz, n_found=err.count(0),
                n_missing=err.count(NONODE), n_error=sum(1 for e in err if e not in (0, NONODE)), n_skipped=skipped,
                consumed=pos)


def classify(paths, payloads, r, session, zk_flags, known_mzxid=None):
    """the table of regk_reconcile_stats over a read `r` -> dict(cls, match, create, update, dup, replace, update_ver,
    replace_ver); raises ValueError naming the smallest record whose reply carries an error other than NONODE"""
    want = session if zk_flags == 1 else 0
    bad = [i for i, e in enumerate(r["err"]) if e not in (0, NONODE)]
    if bad:
        raise ValueError("record %d" % bad[0])
    first, cls, match = {}, [], []
    for i, (p, d) in enumerate(zip(paths, payloads)):
        f = first.setdefault(p, i)
        match.append(f if r["err"][f] == 0 else NO_MATCH)
        if f != i:
            cls.append(DUP)
        elif r["err"][i] == NONODE:
            cls.append(CREATE)
        elif r["owner"][i] != want:
            cls.append(REPLACE)
        elif r["data_length"][i] != len(d) or (known_mzxid is not None and r["mzxid"][i] != known_mzxid[i]):
            cls.append(UPDATE)
        else:
            cls.append(SAME)
    pick = lambda c: [i for i, x in enumerate(cls) if x == c]
    out = dict(cls=cls, match=match, create=pick(CREATE), update=pick(UPDATE), dup=pick(DUP), replace=pick(REPLACE))
    out["update_ver"] = [r["version"][i] for i in out["update"]]
    out["replace_ver"] = [r["version"][i] for i in out["replace"]]
    return out
