"""TEST INFRASTRUCTURE: a restatement of regk_walk_resolve's identity and reuse rules (include/regk.h) on top of
walk_watch_util's model and driver, and registry-shaped random scripts.

Identity: each snapshot node's index at the last successful walk resolve, or None.  A node a plain level appends has
none; a refresh-level getData with err 0 takes it only when the data bytes differ; it moves with its node when the
removed nodes are dropped; walk_start clears it.  Reuse: full when there was no resolve since the start or its default
TTLs differ; otherwise a HOST_A section is copied when its node has an identity, and a service child's lines when the
child and its service both have one.  copied_bytes is predicted from resolve_util.resolve's sections of single nodes
and of (service, child) pairs: a line depends on nothing else."""
import resolve_util as rv
import walk_setwatches_util as ws
import walk_watch_util as ww
from test_resolve_cpu import host, service


class IdentMixin:
    """the identity bookkeeping, mixed into a walk model (walk_watch_util.Model or walk_setwatches_util.Model)"""

    def start(self, roots):
        super().start(roots)
        self.ident, self.last = [], None

    def _drop_removed(self, replaced=None):
        keep = [j for j in range(len(self.nodes)) if not self.marks[j] & ww.REMOVED]
        ident = []
        for j in keep:
            i = self.ident[j]
            if replaced and j in replaced and replaced[j][0] != self.nodes[j][1]:
                i = None
            ident.append(i)
        super()._drop_removed(replaced)
        self.ident = ident

    def read(self, stream):
        r = super().read(stream)
        self.ident += [None] * (len(self.nodes) - len(self.ident))
        return r

    def predict(self, dh, ds):
        """-> (full, n_fresh, copied_bytes) of a walk resolve of the snapshot as it stands"""
        m = len(self.nodes)
        if self.last != (dh, ds):
            return 1, m, 0
        return 0, sum(1 for i in self.ident if i is None), copied_bytes(self.pairs(), self.ident, dh, ds)

    def pairs(self):
        return [(n[0], n[1]) for n in self.nodes]

    def resolved(self, dh, ds):
        """a successful walk resolve"""
        self.ident, self.last = list(range(len(self.nodes))), (dh, ds)


class Model(IdentMixin, ww.Model):
    pass


class SwModel(IdentMixin, ws.Model):
    pass


class Driver(ww.Driver):
    def __init__(self, zk, roots, rng, lib=None):
        super().__init__(zk, roots, rng, lib)
        self.model = Model()


class SwDriver(ws.Driver):
    def __init__(self, zk, roots, rng, lib=None):
        super().__init__(zk, roots, rng, lib)
        self.model = SwModel()


def host_a_bytes(node, dh, ds):
    r = rv.resolve([node], dh, ds)
    return len(r["sections"][0][0]) if r["q_kind"] == [rv.HOST_A] else 0


def child_bytes(svc, child, dh, ds):
    """the bytes of child's A line, SRV lines and additional line under svc (0: not its child)"""
    r = rv.resolve([svc, child], dh, ds)
    if r["q_kind"][:2] != [rv.SERVICE_A, rv.SERVICE_SRV] or r["q_node"][:2] != [0, 0] or not r["sections"][0][0]:
        return 0
    return len(r["sections"][0][0]) + len(r["sections"][1][0]) + len(r["sections"][1][1])


def copied_bytes(nodes, ident, dh, ds):
    index = {p: j for j, (p, _) in enumerate(nodes)}
    total = 0
    for c, node in enumerate(nodes):
        if ident[c] is None:
            continue
        total += host_a_bytes(node, dh, ds)
        path = node[0]
        s = index.get(path[:path.rfind(b"/")]) if path.rfind(b"/") > 0 else None
        if s is not None and ident[s] is not None:
            total += child_bytes(nodes[s], node, dh, ds)
    return total


# ---- registry-shaped trees and mutations ----

TYPES = [b"redis_host", b"redis_host", b"load_balancer", b"host", b"db_host", b"ops_host", b"rr_host", b"moray_host", b"bogus"]


def inst_data(rng, serial):
    ttl = rng.choice([None, None, 30, 120])
    ports = rng.choice([None, None, [6379], [80, 443], []])
    return host(rng.choice(TYPES), b"10.%d.%d.%d" % (serial // 65536 % 256, serial // 256 % 256, serial % 250 + 1), ttl, ports)


def svc_data(rng):
    return service(b"_http", b"_tcp", rng.choice([80, 8080, 443]), rng.choice([60, 60, 300, None]))


def build_registry(zk, rng, root=b"/r", n_svc=4, n_inst=(0, 1, 3, 6)):
    """services under root, instances under each, some under a directory level between service and instance"""
    zk.create(root, b"", 0, False)
    serial = 0
    for s in range(n_svc):
        sp = root + b"/s%d" % s
        zk.create(sp, svc_data(rng), 0, False)
        for i in range(rng.choice(n_inst)):
            serial += 1
            zk.create(sp + b"/i%d" % serial, inst_data(rng, serial), 0, False)
        if rng.random() < 0.4:
            zk.create(sp + b"/dir", b"", 0, False)
            serial += 1
            zk.create(sp + b"/dir/i%d" % serial, inst_data(rng, serial), 0, False)


class RegistryMutator:
    """instances added and deleted; an instance's address, ports or ttl changed; data rewritten with identical bytes;
    a service's ttl or port changed; a service turned into a non-record and back; delete-and-recreate with the same
    data"""

    def __init__(self, zk, root, rng):
        self.zk, self.root, self.rng, self.serial = zk, root, rng, 10 ** 5

    def _nodes(self):
        return [p for p in self.zk.nodes if p.startswith(self.root + b"/")]

    def one(self):
        zk, rng = self.zk, self.rng
        nodes = self._nodes()
        svcs = [p for p in nodes if p.count(b"/") == self.root.count(b"/") + 1]
        leaves = [p for p in nodes if not zk.kids.get(p) and p not in svcs]
        self.serial += 1
        r = rng.random()
        if r < 0.2 or not leaves:
            d = rng.choice(svcs + [p for p in nodes if p.endswith(b"/dir")])
            zk.create(d + b"/n%d" % self.serial, inst_data(rng, self.serial), 0, False)
        elif r < 0.35:
            zk.delete(rng.choice(leaves))
        elif r < 0.5:
            zk.set_data(rng.choice(leaves), inst_data(rng, self.serial))
        elif r < 0.65:
            p = rng.choice(nodes)
            zk.set_data(p, zk.nodes[p].data)
        elif r < 0.75:
            zk.set_data(rng.choice(svcs), svc_data(rng))
        elif r < 0.85:
            p = rng.choice(svcs)
            zk.set_data(p, b"{}" if zk.nodes[p].data.startswith(b"{\"type\":\"service\"") else svc_data(rng))
        else:
            p = rng.choice(leaves)
            data = zk.nodes[p].data
            zk.delete(p)
            zk.create(p, data, 0, False)

    def some(self, n):
        for _ in range(n):
            self.one()

    def in_flight(self, p):
        return lambda k: self.one() if self.rng.random() < p else None


def script(rng, check, rounds=5, n_svc=4, churn=4, flight=0.05, lib=None):
    """a registry-shaped script: the watched walk, then rounds of mutation, events and refresh; check(driver, phase)
    is called after the start, after each round's events (removed nodes still in the snapshot) and after each refresh,
    and after settling -> the Driver"""
    zk = ww.WalkZooKeeper()
    build_registry(zk, rng, b"/r", n_svc)
    d = Driver(zk, [b"/r"], rng, lib)
    mut = RegistryMutator(zk, b"/r", rng)
    d.start()
    check(d, "start")
    for _ in range(rounds):
        mut.some(rng.randrange(churn + 1))
        d.feed(zk.take_events(d.SESSION))
        if rng.random() < 0.3:
            check(d, "events")
        d.refresh(mut.in_flight(flight))
        check(d, "refresh")
    d.settle()
    check(d, "settled")
    assert d.snapshot_set() == zk.subtree([b"/r"])
    return d


def struct_layout(header):
    """the field names of regk_walk_answers, in order, read from include/regk.h"""
    body = header.split("typedef struct regk_walk_answers {")[1].split("} regk_walk_answers;")[0]
    fields = []
    for line in body.splitlines():
        line = line.split("/*")[0].strip().rstrip(";")
        if line:
            fields += [f.strip() for f in line.split(None, 1)[1].split(",")]
    return fields
