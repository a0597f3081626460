"""Independent restatement of regk_jute_requests(REGK_ZK_GETDATA) and of regk_read_replies, for the tests: a
GetDataRequest frame builder, a reply builder that answers parsed getData frames from the ZooKeeper model of
reconcile_owned_util, and a sequential reader of the reply stream.  The layouts follow zookeeper.jute (RequestHeader,
GetDataRequest, ReplyHeader, GetDataResponse, Stat; all integers big endian).  PARITY UNPINNED: they are pinned against a
frame worked out by hand from those definitions, not against a server."""
import struct

import reconcile_owned_util as ou

OP_GETDATA = 4
NOTIFY_XID, PING_XID = -1, -2
ZOK, NONODE = ou.ZOK, ou.NONODE

# refusal codes, as regk_replies.cuh numbers them
OK, TRUNC, BAD_LEN, NEG_XID, XID_RANGE, ERR_BODY, SUCC_LEN, NEG_DATA, STAT_LEN, ORDER = range(10)


def wrap(x):
    return (x + 2 ** 31) % 2 ** 32 - 2 ** 31


def getdata_frames(paths, xid_base=1):
    """len | RequestHeader{xid_base + i, 4} | GetDataRequest{path i, watch = false}, back to back"""
    out = []
    for i, p in enumerate(paths):
        body = struct.pack(">ii", wrap(xid_base + i), OP_GETDATA) + struct.pack(">i", len(p)) + p + b"\x00"
        out.append(struct.pack(">i", len(body)) + body)
    return b"".join(out)


def parse_getdata(frame_bytes):
    """getData frames -> [(xid, path)]"""
    b, k, out = bytes(frame_bytes), 0, []
    while k < len(b):
        ln, xid, op, pl = struct.unpack_from(">iiii", b, k)
        assert op == OP_GETDATA and ln == 13 + pl and b[k + 16 + pl] == 0
        out.append((xid, b[k + 16:k + 16 + pl]))
        k += 4 + ln
    return out


def stat(version=0, owner=0, data_len=0, children=0, seed=0):
    """a Stat record: deterministic zxids and times from `seed`"""
    z = 0x100000000 + 17 * seed
    return struct.pack(">qqqqiiiqiiq", z, z + 5, 1_700_000_000_000 + seed, 1_700_000_000_500 + seed, version, 3, 0, owner,
                       data_len, children, z + 9)


def success(xid, data, version=0, owner=0, children=0, seed=0, null=False, zxid=None):
    """a GetDataResponse reply frame; null=True sends data length -1 (the data must then be empty)"""
    assert not (null and data)
    body = struct.pack(">iqi", xid, 0x200000000 + seed if zxid is None else zxid, ZOK)
    body += struct.pack(">i", -1 if null else len(data)) + data + stat(version, owner, len(data), children, seed)
    return struct.pack(">i", len(body)) + body


def error(xid, err, zxid=7):
    body = struct.pack(">iqi", xid, zxid, err)
    return struct.pack(">i", len(body)) + body


def notification(path=b"/x", typ=3, state=3):
    """a WatcherEvent (xid -1)"""
    body = struct.pack(">iqi", NOTIFY_XID, -1, 0) + struct.pack(">iii", typ, state, len(path)) + path
    return struct.pack(">i", len(body)) + body


def ping():
    return error(PING_XID, 0, zxid=-1)


def replies(zk, frame_bytes, errors=None, null=(), extra=None, trailing=b""):
    """answer every getData frame from the model `zk` (an ou.ZooKeeper): success with the node's data and Stat, NONODE
    when it has no such node.  errors = {record: err} replaces record k's reply by an error reply; null = the records
    whose (empty) data goes out as length -1; extra = {record: bytes} inserts frames (notifications, pings) before
    record k's reply (record n: after the last one); trailing is appended."""
    errors, extra = errors or {}, extra or {}
    out = []
    reqs = parse_getdata(frame_bytes)
    for k, (xid, path) in enumerate(reqs):
        out.append(extra.get(k, b""))
        node = zk.nodes.get(path)
        if k in errors:
            out.append(error(xid, errors[k]))
        elif node is None:
            out.append(error(xid, NONODE))
        else:
            kids = sum(1 for p in zk.nodes if p.startswith(path + b"/") and b"/" not in p[len(path) + 1:])
            out.append(success(xid, node.data, node.version, node.owner, kids, seed=k, null=k in null))
    out.append(extra.get(len(reqs), b""))
    return b"".join(out) + trailing


class Refused(Exception):
    def __init__(self, code, pos, k):
        super().__init__("code %d at byte %d, record %d" % (code, pos, k))
        self.code, self.pos, self.k = code, pos, k


def _i32(b, k):
    return struct.unpack_from(">i", b, k)[0]


def plausible(b, pos, xid_base, n):
    """the plausibility test of regk_read_replies at `pos` -> OK or the refusal code"""
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
    if ln < 20:
        return SUCC_LEN
    d = _i32(b, pos + 20)
    if d < -1:
        return NEG_DATA
    return OK if ln == 88 + max(d, 0) else SUCC_LEN


def read(stream, xid_base, n):
    """the sequential reader: -> dict(err, found, n_found, n_missing, n_error, n_skipped, consumed), where found =
    [(record, data, version, owner)] of every reply with err 0; raises Refused at the first frame that fails"""
    b = bytes(stream)
    pos, k, skipped, err, found = 0, 0, 0, [], []
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
            d = max(_i32(b, pos + 20), 0)
            data = b[pos + 24:pos + 24 + d]
            st = pos + 24 + d
            version, owner, dlen = _i32(b, st + 32), struct.unpack_from(">q", b, st + 44)[0], _i32(b, st + 52)
            if dlen != d:
                raise Refused(STAT_LEN, pos, k)
            found.append((k, data, version, owner))
        err.append(e)
        k += 1
        pos += 4 + ln
    return dict(err=err, found=found, n_found=err.count(0), n_missing=err.count(NONODE),
                n_error=sum(1 for e in err if e not in (0, NONODE)), n_skipped=skipped, consumed=pos)


def snapshot_nodes(paths, r):
    """the snapshot of a read: (node_rec, [(path, data, version, owner)]), the first found reply of every path"""
    seen, rec, nodes = set(), [], []
    for k, data, version, owner in r["found"]:
        if paths[k] not in seen:
            seen.add(paths[k])
            rec.append(k)
            nodes.append((paths[k], data, version, owner))
    return rec, nodes


def device_replies(json_bytes, json_off, xid_base, version, owner, missing=None, chunk=1 << 20):
    """The reply stream to every record of a batch, built on the device with torch: record i's reply is a success
    carrying payload i, version[i] and owner[i] (its Stat otherwise as stat(seed=0) with zxid 0), or NONODE where
    missing[i].  json_off holds uint64 host offsets, json_bytes is a uint8 host array.  Returns a CUDA uint8
    tensor."""
    import numpy as np
    import torch
    n = len(json_off) - 1
    J = np.diff(json_off.astype(np.int64))
    miss = np.zeros(n, bool) if missing is None else np.asarray(missing, bool)
    flen = np.where(miss, 20, 92 + J)
    off = np.zeros(n + 1, np.int64)
    np.cumsum(flen, out=off[1:])
    out = torch.zeros(int(off[-1]), dtype=torch.uint8, device="cuda")
    js = torch.from_numpy(np.ascontiguousarray(json_bytes)).cuda()
    be = lambda v, w: torch.from_numpy(np.ascontiguousarray(np.asarray(v).astype(">i%d" % w)).view(np.uint8).reshape(-1, w))
    tmpl = np.frombuffer(stat(), np.uint8)
    for a in range(0, n, chunk):
        b = min(n, a + chunk)
        m = b - a
        xid = [wrap(xid_base + i) for i in range(a, b)]
        ms = miss[a:b]
        head = np.zeros((m, 24), np.uint8)
        head[:, 0:4] = be(flen[a:b] - 4, 4).numpy()
        head[:, 4:8] = be(np.array(xid, np.int64), 4).numpy()
        head[:, 16:20] = be(np.where(ms, NONODE, 0), 4).numpy()
        head[:, 20:24] = be(J[a:b], 4).numpy()
        st = np.repeat(tmpl[None, :], m, 0)
        st[:, 32:36] = be(version[a:b], 4).numpy()
        st[:, 44:52] = be(owner[a:b], 8).numpy()
        st[:, 52:56] = be(J[a:b], 4).numpy()
        o = torch.from_numpy(off[a:b]).cuda()
        hl = torch.where(torch.from_numpy(ms).cuda(), 20, 24)
        cols = torch.arange(24, device="cuda")
        sel = cols[None, :] < hl[:, None]
        idx = (o[:, None] + cols[None, :])[sel]
        out[idx] = torch.from_numpy(head).cuda()[sel]
        keep = torch.from_numpy(~ms).cuda()
        jl = torch.from_numpy(J[a:b]).cuda()
        jo = torch.from_numpy(json_off[a:b].astype(np.int64)).cuda()
        ok, okl, ojo = o[keep], jl[keep], jo[keep]
        if okl.sum() > 0:
            rep = torch.repeat_interleave(torch.arange(ok.numel(), device="cuda"), okl)
            start = torch.cumsum(okl, 0) - okl
            within = torch.arange(rep.numel(), device="cuda") - start[rep]
            out[ok[rep] + 24 + within] = js[ojo[rep] + within]
        cols = torch.arange(68, device="cuda")
        sidx = (ok + 24 + okl)[:, None] + cols[None, :]
        out[sidx.reshape(-1)] = torch.from_numpy(st[~ms]).cuda().reshape(-1)
    return out
