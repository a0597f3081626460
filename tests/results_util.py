"""Independent restatement of regk_read_results, for the tests: the replies ZooKeeper sends to create, delete, setData
and multi frames (CreateResponse, SetDataResponse's Stat, MultiResponse with typed results or ErrorResults), a server
that answers parsed request frames from the ZooKeeper model of reconcile_owned_util operation by operation, and a
sequential front-to-back reader that turns a reply stream into each entry's outcome.  The layouts follow zookeeper.jute
(ReplyHeader, CreateResponse, SetDataResponse, Stat, MultiHeader, ErrorResponse; integers big endian) and the server's
multi handling.  PARITY UNPINNED: pinned against replies worked out by hand from those definitions, not against a
server."""
import struct

import reconcile_owned_util as ou
import replies_util as ru

OP_CREATE, OP_DELETE, OP_SETDATA, OP_MULTI, OP_REPLACE = 1, 2, 5, 14, 256
RUNTIMEINCONSISTENCY = -2
ZOK, NONODE, NODEEXISTS, BADVERSION, NOTEMPTY = ou.ZOK, ou.NONODE, ou.NODEEXISTS, ou.BADVERSION, ou.NOTEMPTY
DONE, FAILED, ABORTED = 0, 1, 2
notification, ping, wrap, Refused = ru.notification, ru.ping, ru.wrap, ru.Refused

# refusal codes, as regk_results.cuh numbers them
(OK, TRUNC, BAD_LEN, NEG_XID, XID_RANGE, ERR_BODY, SUCC_LEN, ORDER, OP_TYPE, PATH_ECHO, STAT_LEN, ERR_RESULT, ERR_SEQ,
 CLOSE, NO_FAILURE) = range(15)


def _reply(xid, err, body=b"", zxid=0x300000000):
    b = struct.pack(">iqi", xid, zxid, err) + body
    return struct.pack(">i", len(b)) + b


def error(xid, err):
    return _reply(xid, err)


def mh(t, done, err):
    """MultiHeader{type, done, err}"""
    return struct.pack(">ibi", t, 1 if done else 0, err)


def create_body(path):
    return struct.pack(">i", len(path)) + path


def stat_of(node, seed=0):
    return ru.stat(node.version, node.owner, len(node.data), 0, seed)


class Server:
    """Answers request frames from an ou.ZooKeeper, applying them: a single request as the model applies it, a multi
    operation by operation against the state the operations before it left, all or nothing.  Each reply is what the
    server sends: typed results, or (a multi that failed) ErrorResults 0 .. 0, the failing code, -2 .. -2."""

    def __init__(self, zk, session):
        self.zk, self.session = zk, session

    def answer(self, frame, header_err=None):
        xid, ops, multi = ou.parse_frame(frame)
        if header_err is not None:
            return error(xid, header_err)
        if not multi:
            op, path, data, arg = ops[0]
            rc = self.zk._apply(self.zk.nodes, op, path, data, arg, self.session)
            if rc != ZOK:
                return error(xid, rc)
            return _reply(xid, 0, self._result(self.zk.nodes, op, path))
        work = {p: n.copy() for p, n in self.zk.nodes.items()}
        results = []
        for j, (op, path, data, arg) in enumerate(ops):
            rc = self.zk._apply(work, op, path, data, arg, self.session)
            if rc != ZOK:
                codes = [0] * j + [rc] + [RUNTIMEINCONSISTENCY] * (len(ops) - j - 1)
                body = b"".join(mh(-1, False, c) + struct.pack(">i", c) for c in codes)
                return _reply(xid, 0, body + mh(-1, True, -1))
            results.append(mh(op, False, 0) + self._result(work, op, path))
        self.zk.nodes = work
        return _reply(xid, 0, b"".join(results) + mh(-1, True, -1))

    @staticmethod
    def _result(nodes, op, path):
        return create_body(path) if op == OP_CREATE else b"" if op == OP_DELETE else stat_of(nodes[path])

    def replies(self, frame_bytes, frame_off, extra=None, header_err=None):
        """answer every frame in order; extra = {k: bytes} inserts frames before reply k (k = frames: after the last);
        header_err = {k: err} answers frame k with a header-only error and does not apply it"""
        extra, header_err = extra or {}, header_err or {}
        frames = ou.split(frame_bytes, frame_off)
        out = []
        for k, f in enumerate(frames):
            out.append(extra.get(k, b""))
            out.append(self.answer(f, header_err.get(k)))
        out.append(extra.get(len(frames), b""))
        return b"".join(out)


def device_create_replies(path_bytes, path_off, xid_base, err):
    """the replies to single creates of the given paths, built on the device: CreateResponse{path} where err[i] == 0,
    else a header-only error.  Returns a CUDA uint8 tensor."""
    import torch
    dev = "cuda"
    pb = torch.as_tensor(path_bytes).to(dev)
    po = torch.as_tensor(path_off.astype("int64")).to(dev)
    e = torch.as_tensor(err.astype("int64")).to(dev)
    n = e.numel()
    P = po[1:] - po[:-1]
    ok = e == 0
    flen = torch.where(ok, 24 + P, torch.full_like(P, 20))
    off = torch.cumsum(flen, 0) - flen
    total = int(flen.sum())
    xid = (torch.arange(n, device=dev) + xid_base) % 2 ** 32

    def be(x):
        return torch.stack([(x >> s) & 255 for s in (24, 16, 8, 0)], 1)
    head = torch.cat([be(flen - 4), be(xid), be(torch.full_like(P, 3)), be(torch.zeros_like(P)), be(e % 2 ** 32),
                      be(P)], 1).to(torch.uint8)
    out = torch.empty(total, dtype=torch.uint8, device=dev)
    cols = torch.arange(24, device=dev)
    idx = off[:, None] + cols
    mask = cols[None, :] < torch.where(ok, 24, 20)[:, None]
    out[idx[mask]] = head[mask]
    rec = torch.repeat_interleave(torch.arange(n, device=dev), P)
    t = torch.arange(rec.numel(), device=dev) - po[rec]
    keep = ok[rec]
    out[(off[rec] + 24 + t)[keep]] = pb[:rec.numel()][keep]
    return out


class Framing:
    """what a write framing framed: entries e = (path, data length) in frames of `group` (a replace entry is two
    operations), xid_base + k per frame; tol = the code that still counts as done"""

    def __init__(self, op, paths, data_lens=None, xid_base=1, group=0, tol=0):
        self.op, self.paths, self.xid_base, self.tol = op, list(paths), xid_base, tol
        self.data_lens = list(data_lens) if data_lens is not None else [0] * len(self.paths)
        self.multi = op == OP_REPLACE or group != 0
        self.group = max(group, 1)
        self.entries = len(self.paths)
        self.frames = (self.entries + self.group - 1) // self.group

    def span(self, k):
        return k * self.group, min(k * self.group + self.group, self.entries)

    def lens(self, k):
        """(applied length, rolled-back length or None) of frame k's reply"""
        a, b = self.span(k)
        m, P = b - a, sum(len(p) for p in self.paths[a:b])
        if not self.multi:
            return {OP_CREATE: 20 + P, OP_DELETE: 16, OP_SETDATA: 84}[self.op], None
        ok = 25 + {OP_CREATE: 13 * m + P, OP_DELETE: 9 * m, OP_SETDATA: 77 * m, OP_REPLACE: 22 * m + P}[self.op]
        return ok, 25 + 13 * m * (2 if self.op == OP_REPLACE else 1)


def _i32(b, k):
    return struct.unpack_from(">i", b, k)[0]


def plausible(b, pos, fr):
    """results_head at `pos` -> OK or the refusal code"""
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
    k = (xid - fr.xid_base) % 2 ** 32
    if k >= fr.frames:
        return NEG_XID if xid < 0 else XID_RANGE
    if err != 0:
        return OK if ln == 16 else ERR_BODY
    return OK if ln in fr.lens(k) else SUCC_LEN


def _frame_entries(b, pos, fr, k):
    """the outcomes of frame k's entries read front to back -> [(err, cls, version)]; raises Refused at the first fault"""
    ln, herr = _i32(b, pos), _i32(b, pos + 16)
    a, e_end = fr.span(k)
    if herr != 0:
        return [(herr, DONE if fr.tol and herr == fr.tol else FAILED, -1) for _ in range(a, e_end)]
    if not fr.multi:
        p = pos + 20
        if fr.op == OP_CREATE:
            if b[p:p + 4] != struct.pack(">i", len(fr.paths[a])) or b[p + 4:p + 4 + len(fr.paths[a])] != fr.paths[a]:
                raise Refused(PATH_ECHO, p, k)
            return [(0, DONE, 0)]
        if fr.op == OP_SETDATA:
            if _i32(b, p + 52) != fr.data_lens[a]:
                raise Refused(STAT_LEN, p + 52, k)
            return [(0, DONE, _i32(b, p + 32))]
        return [(0, DONE, -1)]
    ok, bad = fr.lens(k)
    rolled = ln == bad and (ln != ok or _i32(b, pos + 20) == -1)
    ops = {OP_REPLACE: [OP_DELETE, OP_CREATE]}.get(fr.op, [fr.op])
    out, q, seen = [], pos + 20, False
    for e in range(a, e_end):
        if not rolled:
            ver = -1
            for op in ops:
                if b[q:q + 9] != mh(op, False, 0):
                    raise Refused(OP_TYPE, q, k)
                q += 9
                if op == OP_CREATE:
                    P = fr.paths[e]
                    if b[q:q + 4 + len(P)] != create_body(P):
                        raise Refused(PATH_ECHO, q, k)
                    q += 4 + len(P)
                    ver = 0
                elif op == OP_SETDATA:
                    if _i32(b, q + 52) != fr.data_lens[e]:
                        raise Refused(STAT_LEN, q + 52, k)
                    ver = _i32(b, q + 32)
                    q += 68
            out.append((0, DONE, ver))
        else:
            fails, own, code = False, 0, 0
            for _ in ops:
                t, done, c = struct.unpack_from(">ibi", b, q)
                if t != -1 or done != 0:
                    raise Refused(OP_TYPE, q, k)
                if _i32(b, q + 9) != c:
                    raise Refused(ERR_RESULT, q, k)
                if seen and c != RUNTIMEINCONSISTENCY:
                    raise Refused(ERR_SEQ, q, k)
                if c != 0 and not seen:
                    seen, fails, code = True, True, c
                own = own or c
                q += 13
            if fails:
                out.append((code, DONE if fr.tol and code == fr.tol else FAILED, -1))
            else:
                out.append((own, ABORTED, -1))
    if b[q:q + 9] != mh(-1, True, -1):
        raise Refused(CLOSE, q, k)
    if rolled and not seen:
        raise Refused(NO_FAILURE, q, k)
    return out


def read(stream, fr, start=0):
    """the sequential reader -> dict(frame_err, err, cls, version, n_skipped, consumed); raises Refused(code, pos, k)"""
    b = bytes(stream)
    pos, k, skipped, ferr, ents = start, 0, 0, [], []
    while k < fr.frames:
        c = plausible(b, pos, fr)
        if c != OK:
            raise Refused(c, pos, k)
        ln, xid = _i32(b, pos), _i32(b, pos + 4)
        if xid in (ru.NOTIFY_XID, ru.PING_XID):
            skipped += 1
            pos += 4 + ln
            continue
        if xid != wrap(fr.xid_base + k):
            raise Refused(ORDER, pos, k)
        ents += _frame_entries(b, pos, fr, k)
        ferr.append(_i32(b, pos + 16))
        k += 1
        pos += 4 + ln
    return dict(frame_err=ferr, err=[e for e, _, _ in ents], cls=[c for _, c, _ in ents], version=[v for _, _, v in ents],
                n_skipped=skipped, consumed=pos)
