"""Independent restatement of the watched walk (regk_walk_requests with REGK_ZK_WATCH, regk_walk_events,
regk_walk_refresh and the refresh level of regk_read_walk), for the tests: a watch-aware tree server built on
events_util.WatchedZooKeeper that also serves getData and arms its data watch, a sequential model of the library's
walk state (snapshot, marks, frontier, level_off) node for node in the order include/regk.h states, and a driver that
runs rounds of mutation, notification and refresh against both, with mutations landing while a level is in flight.
PARITY UNPINNED: the server's watch rules as events_util restates them, not a server."""
import children_util as cu
import events_util as ev
import reconcile_owned_util as ou
import replies_util as ru

OP_GETDATA, OP_GETCHILDREN = 4, 8
NONODE, wrap = ru.NONODE, ru.wrap
PENDING, REMOVED = 1, 2
NO_NODE = 2 ** 64 - 1


class WalkZooKeeper(ev.WatchedZooKeeper):
    """WatchedZooKeeper with getData (op 4, arming the data watch of a node that exists) and a child index, so a
    listing costs its children rather than the whole tree.  Deletes keep the server's NOTEMPTY check."""

    def __init__(self):
        super().__init__()
        self.kids = {b"/": []}

    def _children(self, nodes, path):
        return bool(self.kids.get(path))

    def create(self, path, data, session, ephemeral=False):
        rc = super().create(path, data, session, ephemeral)
        if rc == ou.ZOK:
            self.kids[path] = []
            self.kids[ou.parent(path)].append(path[path.rindex(b"/") + 1:])
        return rc

    def delete(self, path, version=-1):
        rc = super().delete(path, version)
        if rc == ou.ZOK:
            del self.kids[path]
            self.kids[ou.parent(path)].remove(path[path.rindex(b"/") + 1:])
        return rc

    def serve(self, frame_bytes, session, during=None):
        """answer a walk framing in order; during(k) runs after reply k (a mutation while the level is in flight), and
        every notification a mutation fires goes into the stream where it fires -> the session's bytes"""
        out = [self.take_events(session)]
        for k, (xid, op, path, watch) in enumerate(ev.parse_reads(frame_bytes)):
            node = self.nodes.get(path)
            if node is None:
                out.append(ru.error(xid, NONODE))
            elif op == OP_GETDATA:
                if watch:
                    self.data_w.setdefault(session, set()).add(path)
                out.append(ru.success(xid, node.data, node.version, node.owner, len(self.kids[path]), seed=k))
            elif op == OP_GETCHILDREN:
                if watch:
                    self.child_w.setdefault(session, set()).add(path)
                out.append(cu.success(xid, list(self.kids[path])))
            else:
                raise ValueError("only getData and getChildren are served")
            if during:
                during(k)
            out.append(self.take_events(session))
        return b"".join(out)

    def subtree(self, roots):
        """{(path, data, version, owner)} of every node at or under a root"""
        return {(p, n.data, n.version, n.owner) for p, n in self.nodes.items()
                if any(p == r or p.startswith(r + b"/") for r in roots)}


def walk_frames(paths, xid_base, watch):
    """the two-section framing: getData per node, then getChildren per node"""
    f = len(paths)
    return ev.read_frames(OP_GETDATA, paths, xid_base, watch) + ev.read_frames(OP_GETCHILDREN, paths, wrap(xid_base + f), watch)


class Model:
    """the walk state of one context: nodes [(path, data, version, owner)], marks, level_off, frontier (paths; with
    fnode, the snapshot node of each frontier node, on a refresh level), and the watched / refreshed / framing state.
    parent_rule = False leaves out NodeDeleted's parent rule, to show what the rule is for."""

    parent_rule = True

    def start(self, roots):
        self.nodes, self.marks, self.level_off = [], [], [0]
        self.frontier, self.fnode = list(roots), None
        self.watched, self.refreshed, self.framed, self.framed_watch, self.xid = True, False, False, False, 0

    def requests(self, xid_base, watch):
        self.framed, self.framed_watch, self.xid = True, watch, xid_base
        return walk_frames(self.frontier, xid_base, watch)

    def counts(self):
        return (sum(1 for mk in self.marks if mk == PENDING), sum(1 for mk in self.marks if mk & REMOVED))

    def _filter(self, listing, skip_removed):
        held = {self.nodes[j][0] for j in range(len(self.nodes)) if not (skip_removed and self.marks[j] & REMOVED)}
        return [p for p in listing if p not in held]

    def _drop_removed(self, replaced=None):
        replaced = replaced or {}
        keep = [j for j in range(len(self.nodes)) if not self.marks[j] & REMOVED]
        self.nodes = [(self.nodes[j][0],) + replaced[j] if j in replaced else self.nodes[j] for j in keep]
        self.marks = [self.marks[j] & PENDING for j in keep]

    def read(self, stream):
        """regk_read_walk: -> the level's counts (as regk_walk reports them); raises ru.Refused as the library refuses"""
        f, xb, paths = len(self.frontier), self.xid, self.frontier
        r1 = ru.read(stream, xb, f)
        r2 = cu.read(stream, wrap(xb + f), f, start=r1["consumed"])
        listing = [paths[k] + b"/" + n for k in range(f) for n in r2["names"][k]]
        if self.fnode is not None:                      # a refresh level
            found = {k: (data, version, owner) for k, data, version, owner in r1["found"]}
            replaced = {}
            for k, j in enumerate(self.fnode):
                if r1["err"][k] == 0:
                    replaced[j] = found[k]
                elif r1["err"][k] == NONODE:
                    self.marks[j] |= REMOVED
            nxt = self._filter(listing, True)
            self._drop_removed(replaced)
            self.level_off = [len(self.nodes)]
        else:
            nxt = self._filter(listing, False) if self.refreshed else listing
            for k, data, version, owner in r1["found"]:
                self.nodes.append((paths[k], data, version, owner))
                self.marks.append(0)
            self.level_off.append(len(self.nodes))
        self.watched = self.watched and self.framed_watch
        self.frontier, self.fnode, self.framed = nxt, None, False
        return dict(level=len(self.level_off) - 1, m=len(self.nodes), n_frontier=len(nxt), n_found=r1["n_found"],
                    n_missing=r1["n_missing"], n_error=r1["n_error"], n_listed=r2["n_found"],
                    n_list_missing=r2["n_missing"], n_list_error=r2["n_error"], n_children=len(listing),
                    n_skipped=r1["n_skipped"] + r2["n_skipped"], consumed=r2["consumed"])

    def events(self, stream, start=0, xid_base=0, n_xids=0):
        """regk_walk_events: -> dict(events [(pos, type, state, zxid, node)], counts); raises ev.Refused"""
        r = ev.read(stream, xid_base, n_xids, start)
        present = {self.nodes[j][0]: j for j in range(len(self.nodes)) if not self.marks[j] & REMOVED}
        out, unmatched, other, pend, gone = [], 0, 0, [], []
        for pos, typ, state, zxid, path in r["events"]:
            j = present.get(path) if typ in (ev.DELETED, ev.DATA_CHANGED, ev.CHILDREN_CHANGED) else None
            if j is None:
                unmatched += 1
            elif typ == ev.DELETED:
                gone.append(j)
                d = path[:max(path.rfind(b"/"), 0)]
                if self.parent_rule and d and d in present:
                    pend.append(present[d])
            else:
                pend.append(j)
            other += typ == ev.NONE or typ >= 5
            out.append((pos, typ, state, zxid, NO_NODE if j is None else j))
        for j in pend:
            self.marks[j] |= PENDING
        for j in gone:
            self.marks[j] |= REMOVED
        n_pending, n_removed = self.counts()
        return dict(events=out, n_events=len(out), n_pings=r["n_pings"], n_replies=r["n_replies"], n_unmatched=unmatched,
                    n_other=other, consumed=r["consumed"], partial=r["partial"], n_pending=n_pending, n_removed=n_removed)

    def refresh(self):
        """regk_walk_refresh -> dict(n_removed, n_kept, n_frontier)"""
        m0 = len(self.nodes)
        self._drop_removed()
        pend = [j for j in range(len(self.nodes)) if self.marks[j] == PENDING]
        self.marks = [0] * len(self.nodes)
        self.frontier = [self.nodes[j][0] for j in pend]
        self.fnode = pend if pend else None
        self.refreshed, self.framed = True, False
        self.level_off = [len(self.nodes)]
        return dict(n_removed=m0 - len(self.nodes), n_kept=len(self.nodes), n_frontier=len(pend))


class Driver:
    """rounds of mutation and refresh over a WalkZooKeeper and a Model; `lib` (optional) is called in lockstep with
    the model: lib.start(roots), lib.requests(xid, watch, frames), lib.read(stream, want), lib.events(stream, start,
    xid_base, n_xids, want), lib.refresh(want), each checking the library against what the model says"""

    SESSION = 0x5EED

    def __init__(self, zk, roots, rng, lib=None):
        self.zk, self.roots, self.rng, self.lib = zk, list(roots), rng, lib
        self.model, self.xid = Model(), 1

    def _next_xid(self, n):
        if any((r - self.xid) % 2 ** 32 < n for r in (2 ** 32 - 1, 2 ** 32 - 2)):
            self.xid = 0
        x, self.xid = self.xid, (self.xid + n) % 2 ** 32
        return wrap(x)

    def feed(self, stream, xid_base=0, n_xids=0):
        """the events of a stream, through the model and the library; sometimes in two pieces cut at a random byte"""
        start = 0
        if stream and self.rng.random() < 0.3:
            want = self._events(stream[:self.rng.randrange(len(stream))], 0, xid_base, n_xids)
            start = want["consumed"]
        want = self._events(stream, start, xid_base, n_xids)
        assert not want["partial"] and want["consumed"] == len(stream)
        return want

    def _events(self, stream, start, xid_base, n_xids):
        want = self.model.events(stream, start, xid_base, n_xids)
        if self.lib:
            self.lib.events(stream, start, xid_base, n_xids, want)
        return want

    def level(self, during=None, watch=True):
        f = len(self.model.frontier)
        xb = self._next_xid(2 * f)
        frames = self.model.requests(xb, watch)
        if self.lib:
            self.lib.requests(xb, watch, frames)
        stream = self.zk.serve(frames, self.SESSION, during)
        want = self.model.read(stream)
        if self.lib:
            self.lib.read(stream, want, self.model)
        if watch:
            self.feed(stream, xb, 2 * f)
        return want

    def levels(self, during=None, watch=True):
        while self.model.frontier:
            self.level(during, watch)

    def start(self, watch=True):
        self.model.start(self.roots)
        if self.lib:
            self.lib.start(self.roots)
        self.levels(watch=watch)

    def refresh(self, during=None):
        want = self.model.refresh()
        if self.lib:
            self.lib.refresh(want, self.model)
        self.levels(during)
        return want

    def settle(self, limit=50):
        """refresh until nothing is pending or removed (the tree no longer changes)"""
        self.feed(self.zk.take_events(self.SESSION))
        for _ in range(limit):
            if self.model.counts() == (0, 0):
                return
            self.refresh()
            self.feed(self.zk.take_events(self.SESSION))
        raise AssertionError("no convergence")

    def snapshot_set(self):
        nodes = self.model.nodes
        assert len({n[0] for n in nodes}) == len(nodes), "a path twice"
        return set(nodes)


def build_tree(zk, rng, root=b"/z", depth=3, fan=(0, 1, 2, 4)):
    """a random tree under root: directories persistent, leaves with data, some ephemeral"""
    zk.create(root, b"", 0, False)
    level = [root]
    for d in range(depth):
        nxt = []
        for p in level:
            for k in range(rng.choice(fan)):
                c = p + b"/n%d_%d" % (d, k)
                zk.create(c, b"v%d" % rng.randrange(1000), 0, False)
                nxt.append(c)
        level = nxt


class Mutator:
    """random mutations of the tree under `roots` (never a root itself): creates, leaf deletes, setData,
    delete-and-recreate"""

    def __init__(self, zk, roots, rng):
        self.zk, self.roots, self.rng, self.serial = zk, list(roots), rng, 0

    def _under(self):
        return [p for p in self.zk.nodes if any(p.startswith(r + b"/") for r in self.roots)]

    def one(self):
        zk, rng = self.zk, self.rng
        nodes = self._under()
        leaves = [p for p in nodes if not zk.kids.get(p)]
        r = rng.random()
        self.serial += 1
        if r < 0.35 or not leaves:
            dirs = [p for p in nodes + self.roots if p in zk.nodes and zk.nodes[p].owner == 0]
            if dirs:
                d = rng.choice(dirs)
                zk.create(d + b"/c%d" % self.serial, b"new%d" % self.serial, self.SESSION_OWNER if rng.random() < 0.3 else 0,
                          rng.random() < 0.3)
        elif r < 0.6:
            zk.delete(rng.choice(leaves))
        elif r < 0.85:
            p = rng.choice(nodes)
            zk.set_data(p, b"set%d" % self.serial)
        else:
            p = rng.choice(leaves)
            eph = zk.nodes[p].owner != 0
            zk.delete(p)
            zk.create(p, b"again%d" % self.serial, self.SESSION_OWNER, eph)

    SESSION_OWNER = 0x1234567890

    def some(self, n):
        for _ in range(n):
            self.one()

    def in_flight(self, p):
        """a `during` callback: after each reply, a mutation with probability p"""
        return lambda k: self.one() if self.rng.random() < p else None


def spent_watch_race(lib=None, parent_rule=True):
    """the race NodeDeleted's parent rule is for: g's child watch is spent (a child created under it), so a refresh
    re-reads g; between g's getData and getChildren replies p is deleted and recreated.  The delete fires only p's
    NodeDeleted (g's child watch is not armed again until g's getChildren), and g's listing shows the new p while the
    old p is still a node, so the new p is filtered out.  -> the Driver after one refresh (not settled); the new p is
    walked only if p's NodeDeleted makes g pending"""
    import random
    zk = WalkZooKeeper()
    for path, data in ((b"/z", b""), (b"/z/g", b"g"), (b"/z/g/p", b"p1"), (b"/z/g/q", b"q1")):
        zk.create(path, data, 0, False)
    d = Driver(zk, [b"/z"], random.Random(0), lib)
    d.model.parent_rule = parent_rule
    d.start()
    zk.create(b"/z/g/c", b"c1", 0, False)                      # spends g's child watch
    assert d.feed(zk.take_events(d.SESSION))["n_pending"] == 1
    fired = []

    def during(k):
        if not fired and k == 0:                               # after g's getData reply, before its getChildren reply
            fired.append(k)
            zk.delete(b"/z/g/p")
            zk.create(b"/z/g/p", b"p2", 0, False)
            assert zk.queue[d.SESSION] == [ev.notification(b"/z/g/p", ev.DELETED, zxid=zk.zxid - 1)]
    assert d.refresh(during)["n_frontier"] == 1
    p = [n[0] for n in d.model.nodes].index(b"/z/g/p")
    assert fired and d.model.nodes[p][1] == b"p1" and d.model.marks[p] & REMOVED   # the old p, marked; the new p unread
    return d


def script(rng, lib=None, rounds=6, depth=3, fan=(0, 1, 2, 4), churn=4, flight=0.05, roots=(b"/z",)):
    """one random mutation script to convergence -> the Driver; asserts the convergence property"""
    zk = WalkZooKeeper()
    for r in roots:
        build_tree(zk, rng, r, depth, fan)
    d = Driver(zk, roots, rng, lib)
    mut = Mutator(zk, roots, rng)
    d.start()
    assert d.snapshot_set() == zk.subtree(roots)
    for _ in range(rounds):
        mut.some(rng.randrange(churn + 1))
        d.feed(zk.take_events(d.SESSION))
        d.refresh(mut.in_flight(flight))
    d.settle()
    assert d.snapshot_set() == zk.subtree(roots)
    return d


def struct_layouts(header):
    """(names of regk_walk_events_out's and regk_walk_refresh_out's fields, in order) read from include/regk.h"""
    out = {}
    for name in ("regk_walk_events_out", "regk_walk_refresh_out"):
        body = header.split("typedef struct %s {" % name)[1].split("} %s;" % name)[0]
        fields = []
        for line in body.splitlines():
            line = line.split("/*")[0].strip().rstrip(";")
            if not line:
                continue
            decl = line.split(None, 1)[1] if not line.startswith("const") else line.split("*", 1)[1]
            fields += [f.strip().lstrip("*").strip() for f in decl.split(",")]
        out[name] = fields
    return out

