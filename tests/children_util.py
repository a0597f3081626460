"""Independent restatement of regk_children_requests and regk_read_children, for the tests: GetChildrenRequest frames,
GetChildrenResponse builders (success with names, null vector, error; notifications and pings from replies_util), a
sequential front-to-back reader of the reply stream, the directory set of a batch, the keep / stale rule, and
list_children over the ZooKeeper model of reconcile_owned_util.  The layouts follow zookeeper.jute (RequestHeader,
GetChildrenRequest, ReplyHeader, GetChildrenResponse; integers big endian).  PARITY UNPINNED: pinned against a request
and a response worked out by hand from those definitions, not against a server."""
import struct

import mkdirp_util
import replies_util as ru

OP_GETCHILDREN = 8
ZOK, NONODE = ru.ZOK, ru.NONODE
KEEP, STALE = 0, 1
notification, ping, wrap = ru.notification, ru.ping, ru.wrap

# refusal codes, as regk_children.cuh numbers them
(OK, TRUNC, BAD_LEN, NEG_XID, XID_RANGE, ERR_BODY, SUCC_LEN, NEG_COUNT, ORDER, ENT_TRUNC, ENT_EMPTY, NAME_SLASH, NAME_NUL,
 NAME_DOT, ENT_END) = range(15)


def getchildren_frames(dirs, xid_base=1):
    """len | RequestHeader{xid_base + k, 8} | GetChildrenRequest{dir k, watch = false}, back to back"""
    out = []
    for k, d in enumerate(dirs):
        body = struct.pack(">ii", wrap(xid_base + k), OP_GETCHILDREN) + struct.pack(">i", len(d)) + d + b"\x00"
        out.append(struct.pack(">i", len(body)) + body)
    return b"".join(out)


def parse_getchildren(frame_bytes):
    """getChildren frames -> [(xid, dir)]"""
    b, k, out = bytes(frame_bytes), 0, []
    while k < len(b):
        ln, xid, op, pl = struct.unpack_from(">iiii", b, k)
        assert op == OP_GETCHILDREN and ln == 13 + pl and b[k + 16 + pl] == 0
        out.append((xid, b[k + 16:k + 16 + pl]))
        k += 4 + ln
    return out


def success(xid, names, zxid=0x200000000):
    body = struct.pack(">iqi", xid, zxid, ZOK) + struct.pack(">i", len(names))
    body += b"".join(struct.pack(">i", len(n)) + n for n in names)
    return struct.pack(">i", len(body)) + body


def null_vector(xid, zxid=0x200000000):
    body = struct.pack(">iqii", xid, zxid, ZOK, -1)
    return struct.pack(">i", len(body)) + body


def error(xid, err, zxid=7):
    return ru.error(xid, err, zxid)


def list_children(zk, d):
    """the names of the children of directory d in the model, in its insertion order"""
    pre = d + b"/"
    return [p[len(pre):] for p in zk.nodes if p.startswith(pre) and b"/" not in p[len(pre):]]


def replies(zk, frame_bytes, errors=None, null=(), extra=None, trailing=b""):
    """answer every getChildren frame from the model: the directory's children, NONODE when it does not exist.
    errors = {k: err} replaces reply k by an error; null = directories whose empty listing goes out as count -1;
    extra = {k: bytes} inserts frames before reply k (k = d: after the last); trailing is appended."""
    errors, extra = errors or {}, extra or {}
    out = []
    reqs = parse_getchildren(frame_bytes)
    for k, (xid, d) in enumerate(reqs):
        out.append(extra.get(k, b""))
        if k in errors:
            out.append(error(xid, errors[k]))
        elif d not in zk.nodes:
            out.append(error(xid, NONODE))
        else:
            kids = list_children(zk, d)
            out.append(null_vector(xid) if k in null and not kids else success(xid, kids))
    out.append(extra.get(len(reqs), b""))
    return b"".join(out) + trailing


Refused = ru.Refused


def _i32(b, k):
    return struct.unpack_from(">i", b, k)[0]


def plausible(b, pos, xid_base, d):
    """children_head at `pos` -> OK or the refusal code"""
    avail = len(b) - pos
    if avail < 4:
        return TRUNC
    ln = _i32(b, pos)
    if ln < 16:
        return BAD_LEN
    if ln + 4 > avail:
        return TRUNC
    xid, err = _i32(b, pos + 4), _i32(b, pos + 16)
    if xid in (ru.NOTIFY_XID, ru.PING_XID):
        return OK
    if (xid - xid_base) % 2 ** 32 >= d:
        return NEG_XID if xid < 0 else XID_RANGE
    if err != 0:
        return OK if ln == 16 else ERR_BODY
    if ln < 20:
        return SUCC_LEN
    c = _i32(b, pos + 20)
    if c < -1:
        return NEG_COUNT
    return OK if ln >= 20 + 5 * max(c, 0) else SUCC_LEN


def entry(b, p, end):
    """children_entry at p with the frame ending at `end` -> (code, name length)"""
    if end - p < 4:
        return ENT_TRUNC, 0
    n = _i32(b, p)
    if n < 1:
        return ENT_EMPTY, 0
    if n + 4 > end - p:
        return ENT_TRUNC, 0
    name = b[p + 4:p + 4 + n]
    for c in name:
        if c == 0x2F:
            return NAME_SLASH, n
        if c == 0:
            return NAME_NUL, n
    if name in (b".", b".."):
        return NAME_DOT, n
    return OK, n


def read(stream, xid_base, d, start=0):
    """the sequential reader: -> dict(err, names (per directory), n_found, n_missing, n_error, n_skipped, consumed);
    raises Refused(code, pos, k) at the first fault"""
    b = bytes(stream)
    pos, k, skipped, err, names = start, 0, 0, [], []
    while k < d:
        c = plausible(b, pos, xid_base, d)
        if c != OK:
            raise Refused(c, pos, k)
        ln, xid, e = _i32(b, pos), _i32(b, pos + 4), _i32(b, pos + 16)
        if xid in (ru.NOTIFY_XID, ru.PING_XID):
            skipped += 1
            pos += 4 + ln
            continue
        if xid != wrap(xid_base + k):
            raise Refused(ORDER, pos, k)
        end = pos + 4 + ln
        kids = []
        if e == 0:
            p = pos + 24
            for _ in range(max(_i32(b, pos + 20), 0)):
                code, n = entry(b, p, end)
                if code != OK:
                    raise Refused(code, p, k)
                kids.append(b[p + 4:p + 4 + n])
                p += 4 + n
            if p != end:
                raise Refused(ENT_END, p, k)
        err.append(e)
        names.append(kids)
        k += 1
        pos = end
    return dict(err=err, names=names, n_found=err.count(0), n_missing=err.count(NONODE),
                n_error=sum(1 for e in err if e not in (0, NONODE)), n_skipped=skipped, consumed=pos)


def dir_set(paths):
    """(listed, unlisted): the distinct parent directories in order of first record - listed [(record, dir)] but "/"
    and directories ZooKeeper rejects, whose first records are unlisted"""
    seen, listed, unlisted = set(), [], []
    for i, p in enumerate(paths):
        d = mkdirp_util.dir_of(p)
        if d in seen:
            continue
        seen.add(d)
        if d in (b"", b"/") or mkdirp_util.zk_rejects(d):
            unlisted.append(i)
        else:
            listed.append((i, d))
    return listed, unlisted


def keep_set(paths):
    """the batch's paths and every component-boundary prefix of every listed directory"""
    keep = set(paths)
    for _, d in dir_set(paths)[0]:
        keep.update(mkdirp_util.ancestors(d))
    return keep


def classify(paths, r):
    """a read's listing -> (listing paths, child_off, cls, stale)"""
    listed, _ = dir_set(paths)
    keep = keep_set(paths)
    listing, off = [], [0]
    for (_, d), kids in zip(listed, r["names"]):
        listing += [d + b"/" + n for n in kids]
        off.append(len(listing))
    cls = [KEEP if e in keep else STALE for e in listing]
    return listing, off, cls, [e for e, c in enumerate(cls) if c == STALE]
