"""Independent restatement of regk_reconcile_owned and of the frames regk_reconcile_requests builds after it (replace
multi transactions, observed versions), and a small in-memory ZooKeeper that applies request frames with the server's
checks, for the tests."""
import struct

from oracle import pyoracle
import reconcile_util as ru

SAME, CREATE, UPDATE, DUP, REPLACE = 0, 1, 2, 3, 4
KEEP, DELETE = ru.KEEP, ru.DELETE
NO_MATCH = ru.NO_MATCH
OP_CREATE, OP_DELETE, OP_SETDATA, OP_MULTI = 1, 2, 5, 14

# ZooKeeper KeeperException codes
ZOK, NONODE, BADVERSION, NOCHILDRENFOREPHEMERALS, NODEEXISTS, NOTEMPTY = 0, -101, -103, -108, -110, -111


def reconcile_owned(paths, payloads, nodes, session, zk_flags):
    """nodes = [(path, data, version, owner)] -> ru.reconcile's dict plus `replace`, and the version of each update,
    delete and replace entry's node (`update_ver`, `delete_ver`, `replace_ver`)"""
    r = ru.reconcile(paths, payloads, [(p, d) for p, d, _, _ in nodes])
    want = session if zk_flags == 1 else 0
    cls = list(r["cls"])
    for i, c in enumerate(cls):
        if c in (SAME, UPDATE) and nodes[r["match"][i]][3] != want:
            cls[i] = REPLACE
    pick = lambda c: [i for i, x in enumerate(cls) if x == c]
    r.update(cls=cls, update=pick(UPDATE), replace=pick(REPLACE))
    r["update_ver"] = [nodes[r["match"][i]][2] for i in r["update"]]
    r["replace_ver"] = [nodes[r["match"][i]][2] for i in r["replace"]]
    r["delete_ver"] = [nodes[j][2] for j in r["delete"]]
    return r


def _wrap(x):
    return (x + 2 ** 31) % 2 ** 32 - 2 ** 31


def _mh(op, done=False):
    return struct.pack(">i", op) + (b"\x01" if done else b"\x00") + struct.pack(">i", -1)


def _frame(xid, op, body):
    b = struct.pack(">ii", xid, op) + body
    return struct.pack(">i", len(b)) + b


def versioned_frames(op, items, xid_base=1, group=0):
    """delete / setData over [(path, data, version)], each request with its own version"""
    if group == 0:
        return b"".join(pyoracle.jute_request(op, p, d, _wrap(xid_base + k), 1, v) for k, (p, d, v) in enumerate(items))
    out = []
    for k in range(0, len(items), group):
        body = b"".join(_mh(op) + pyoracle.jute_body(op, p, d, 1, v) for p, d, v in items[k:k + group])
        out.append(_frame(_wrap(xid_base + k // group), OP_MULTI, body + _mh(-1, True)))
    return b"".join(out)


def replace_frames(items, xid_base=1, group=0, zk_flags=1):
    """[(path, data, version)] -> multi transactions of max(group, 1) entries: delete at the version, then create"""
    g = max(group, 1)
    out = []
    for k in range(0, len(items), g):
        body = b"".join(_mh(OP_DELETE) + pyoracle.jute_body(OP_DELETE, p, b"", zk_flags, v) +
                        _mh(OP_CREATE) + pyoracle.jute_body(OP_CREATE, p, d, zk_flags) for p, d, v in items[k:k + g])
        out.append(_frame(_wrap(xid_base + k // g), OP_MULTI, body + _mh(-1, True)))
    return b"".join(out)


# ---------------------------------------------------------------------------------------------- request parsing --

class _Reader:
    def __init__(self, b):
        self.b, self.k = b, 0

    def int(self):
        v = struct.unpack_from(">i", self.b, self.k)[0]
        self.k += 4
        return v

    def long(self):
        v = struct.unpack_from(">q", self.b, self.k)[0]
        self.k += 8
        return v

    def bool(self):
        self.k += 1
        return self.b[self.k - 1] != 0

    def buf(self):
        n = self.int()
        self.k += max(n, 0)
        return b"" if n < 0 else bytes(self.b[self.k - n:self.k])


def _op(r, op):
    """one request record -> (op, path, data, version or flags)"""
    path = r.buf()
    if op == OP_CREATE:
        data = r.buf()
        for _ in range(r.int()):
            r.int(), r.buf(), r.buf()
        return (op, path, data, r.int())
    if op == OP_DELETE:
        return (op, path, b"", r.int())
    if op == OP_SETDATA:
        data = r.buf()
        return (op, path, data, r.int())
    raise ValueError("op %d" % op)


def parse_frame(frame):
    """one length-prefixed frame -> (xid, [(op, path, data, version or flags)], multi)"""
    r = _Reader(frame)
    assert r.int() == len(frame) - 4
    xid, op = r.int(), r.int()
    if op != OP_MULTI:
        ops = [_op(r, op)]
    else:
        ops = []
        while True:
            t, done, err = r.int(), r.bool(), r.int()
            assert err == -1
            if done:
                assert t == -1
                break
            ops.append(_op(r, t))
    assert r.k == len(frame)
    return xid, ops, op == OP_MULTI


def split(frame_bytes, frame_off):
    b = bytes(frame_bytes)
    return [b[int(frame_off[k]):int(frame_off[k + 1])] for k in range(len(frame_off) - 1)]


# ------------------------------------------------------------------------------------------------ the ZooKeeper --

class Node:
    def __init__(self, data, owner):
        self.data, self.version, self.owner = data, 0, owner

    def copy(self):
        n = Node(self.data, self.owner)
        n.version = self.version
        return n


def parent(path):
    k = path.rindex(b"/")
    return b"/" if k == 0 else path[:k]


class ZooKeeper:
    """Nodes keyed by path; "/" always exists.  create / delete / setData / multi with the server's checks:
    NODEEXISTS, NONODE (a missing parent included), BADVERSION (-1 = any), NOTEMPTY, NOCHILDRENFOREPHEMERALS; an
    ephemeral node is owned by the session that created it; setData bumps the version; a multi applies every operation
    against the state the operations before it left, and all of them or none."""

    def __init__(self):
        self.nodes = {}

    def _children(self, nodes, path):
        pre = path + b"/"
        return any(p.startswith(pre) for p in nodes)

    def _apply(self, nodes, op, path, data, arg, session):
        if op == OP_CREATE:
            if path in nodes:
                return NODEEXISTS
            par = parent(path)
            if par != b"/" and par not in nodes:
                return NONODE
            if par != b"/" and nodes[par].owner != 0:
                return NOCHILDRENFOREPHEMERALS
            nodes[path] = Node(data, session if arg & 1 else 0)
            return ZOK
        n = nodes.get(path)
        if n is None:
            return NONODE
        if arg != -1 and arg != n.version:
            return BADVERSION
        if op == OP_DELETE:
            if self._children(nodes, path):
                return NOTEMPTY
            del nodes[path]
        else:
            n.data = data
            n.version = n.version + 1 if n.version < 2 ** 31 - 1 else -2 ** 31
        return ZOK

    def create(self, path, data, session, ephemeral=True):
        return self._apply(self.nodes, OP_CREATE, path, data, 1 if ephemeral else 0, session)

    def delete(self, path, version=-1):
        return self._apply(self.nodes, OP_DELETE, path, b"", version, 0)

    def set_data(self, path, data, version=-1):
        return self._apply(self.nodes, OP_SETDATA, path, data, version, 0)

    def apply_frame(self, frame, session):
        """-> ZOK or the first error; a multi that fails leaves every node as it was"""
        _, ops, multi = parse_frame(frame)
        work = {p: n.copy() for p, n in self.nodes.items()} if multi else self.nodes
        for op, path, data, arg in ops:
            rc = self._apply(work, op, path, data, arg, session)
            if rc != ZOK:
                return rc
        self.nodes = work
        return ZOK

    def apply_frames(self, frame_bytes, frame_off, session):
        return [self.apply_frame(f, session) for f in split(frame_bytes, frame_off)]
