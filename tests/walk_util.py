"""Independent restatement of the registry walk (regk_walk_start / regk_walk_requests / regk_read_walk), for the tests: a
ZooKeeper tree model (path -> data, version, owner, with an ordered child list), a parser of the library's two-section
request buffer that checks op, xid and path, replies built with the builders of replies_util and children_util, knobs
for races, error codes, shuffled listings and interleaved notifications and pings, a sequential reader of one level,
and the breadth-first walk of a tree.  PARITY UNPINNED: the layouts are zookeeper.jute's, as in those modules."""
import struct

import children_util as cu
import mkdirp_util
import reader_fuzz_util as fz
import replies_util as ru

OP_GETDATA, OP_GETCHILDREN = ru.OP_GETDATA, cu.OP_GETCHILDREN
NONODE, wrap = ru.NONODE, ru.wrap


class Tree:
    """path -> [data, version, owner]; kids[path] = child names in creation order"""

    def __init__(self):
        self.nodes, self.kids = {}, {}

    def add(self, path, data=b"", version=0, owner=0):
        assert path not in self.nodes
        self.nodes[path] = [data, version, owner]
        self.kids.setdefault(path, [])
        d = path[:path.rfind(b"/")] or b"/"
        self.kids.setdefault(d, []).append(path[path.rfind(b"/") + 1:])

    def remove(self, path):
        """the node and its subtree"""
        for name in list(self.kids.get(path, [])):
            self.remove(path + b"/" + name)
        del self.nodes[path]
        self.kids.pop(path, None)
        d = path[:path.rfind(b"/")] or b"/"
        self.kids[d].remove(path[path.rfind(b"/") + 1:])

    def children(self, path):
        return list(self.kids.get(path, []))


def bfs(tree, roots):
    """the walk of an unchanging tree: (nodes [(path, data, version, owner)], level_off)"""
    nodes, off, frontier = [], [0], list(roots)
    while frontier:
        nxt = []
        for p in frontier:
            if p in tree.nodes:
                nodes.append((p,) + tuple(tree.nodes[p]))
                nxt += [p + b"/" + n for n in tree.children(p)]
        off.append(len(nodes))
        frontier = nxt
    return nodes, off


def parse_requests(frame_bytes, xid_base):
    """the two-section buffer -> the frontier's paths; asserts op, xid, layout and that both sections frame one list"""
    b, k, out = bytes(frame_bytes), 0, []
    while k < len(b):
        ln, xid, op, pl = struct.unpack_from(">iiii", b, k)
        assert ln == 13 + pl and b[k + 16 + pl] == 0
        out.append((op, xid, b[k + 16:k + 16 + pl]))
        k += 4 + ln
    assert k == len(b) and len(out) % 2 == 0
    f = len(out) // 2
    for i, (op, xid, _) in enumerate(out):
        assert op == (OP_GETDATA if i < f else OP_GETCHILDREN) and xid == wrap(xid_base + i)
    paths = [p for _, _, p in out[:f]]
    assert [p for _, _, p in out[f:]] == paths
    return paths


def first_xid(frame_bytes):
    """the xid base of a framing: its first frame's xid"""
    return struct.unpack_from(">i", bytes(frame_bytes), 4)[0]


def answer(tree, frame_bytes, xid_base, rng=None, gd_errors=None, gc_errors=None, between=None, shuffle=False, noise=0,
           null=False, trailing=b""):
    """the reply stream to one framing, answered from `tree`: gd_errors / gc_errors = {node: err} replace a reply by an
    error; between(tree, paths) runs after the getData replies (a race: the getChildren replies see its changes);
    shuffle lists children in a random order; noise inserts that many notifications and pings anywhere; null sends an
    empty data as length -1 and an empty listing as count -1 for every other node"""
    gd_errors, gc_errors = gd_errors or {}, gc_errors or {}
    paths = parse_requests(frame_bytes, xid_base)
    f = len(paths)
    frames = []
    for i, p in enumerate(paths):
        xid = wrap(xid_base + i)
        n = tree.nodes.get(p)
        if i in gd_errors:
            frames.append(ru.error(xid, gd_errors[i]))
        elif n is None:
            frames.append(ru.error(xid, NONODE))
        else:
            frames.append(ru.success(xid, n[0], n[1], n[2], len(tree.children(p)), seed=i, null=null and not n[0] and i % 2 == 0))
    if between:
        between(tree, paths)
    for i, p in enumerate(paths):
        xid = wrap(xid_base + f + i)
        if i in gc_errors:
            frames.append(cu.error(xid, gc_errors[i]))
        elif p not in tree.nodes:
            frames.append(cu.error(xid, NONODE))
        else:
            kids = tree.children(p)
            if shuffle:
                rng.shuffle(kids)
            frames.append(cu.null_vector(xid) if null and not kids and i % 2 == 0 else cu.success(xid, kids))
    if noise:
        frames = fz.interleave(frames, rng, fz.noise(rng, paths, noise))
    return b"".join(frames) + trailing


def read_level(stream, paths, xid_base):
    """the sequential reader of one level (replies_util.read on the getData section, children_util.read on the
    getChildren section from its end) -> dict(nodes, frontier, counts...); raises ru.Refused at the first fault"""
    f = len(paths)
    r1 = ru.read(stream, xid_base, f)
    r2 = cu.read(stream, wrap(xid_base + f), f, start=r1["consumed"])
    nodes = [(paths[k], data, version, owner) for k, data, version, owner in r1["found"]]
    frontier = [paths[k] + b"/" + n for k in range(f) for n in r2["names"][k]]
    return dict(nodes=nodes, frontier=frontier, n_found=r1["n_found"], n_missing=r1["n_missing"], n_error=r1["n_error"],
                n_listed=r2["n_found"], n_list_missing=r2["n_missing"], n_list_error=r2["n_error"],
                n_children=len(frontier), n_skipped=r1["n_skipped"] + r2["n_skipped"], consumed=r2["consumed"])


def root_error(roots):
    """the smallest bad root of regk_walk_start and why ("rejects", "/", "equals", "under"), or None"""
    first = {}
    for i, r in enumerate(roots):
        first.setdefault(r, i)
    for i, r in enumerate(roots):
        if r == b"/":
            return i, "/"
        if not r or mkdirp_util.zk_rejects(r):
            return i, "rejects"
        if first[r] != i:
            return i, "equals"
        if any(r[t] == 0x2F and r[:t] in first for t in range(1, len(r))):
            return i, "under"
    return None


def readme_tree():
    """the reference README's authcache example (README.md:502-536): the service record at
    /us/joyent/emy-10/authcache and its two redis_host instances, in this library's canonical payload forms"""
    from test_resolve_cpu import AC1, AC2, host, service
    t = Tree()
    t.add(b"/us")
    t.add(b"/us/joyent")
    t.add(b"/us/joyent/emy-10")
    t.add(b"/us/joyent/emy-10/authcache", service(b"_redis", b"_tcp", 6379, 60), version=2)
    for name, addr in ((AC1, b"10.99.99.29"), (AC2, b"10.99.99.30")):
        t.add(b"/us/joyent/emy-10/authcache/" + name, host(b"redis_host", addr, None, [6379]), version=1,
              owner=0x100000001)
    return t
