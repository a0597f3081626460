"""regk_resolve on the GPU, bit for bit against the restatement in resolve_util: the reference README's scenarios,
random mixed snapshots (directories, non-canonical and escaped payloads, every class, services without children,
host records under host records and directories, a service under a service, ports: [], absent ttls) from host and
device snapshots with and without REGK_OUT_DEVICE, the refusals, the getData pipeline straight from read_replies'
device snapshot, and a fleet of a million host records under 1 000 services."""
import random

import numpy as np
import pytest

import replies_util as ru
import resolve_util as rv
from test_reconcile import _dev, device_snapshot
from test_resolve_cpu import check_readme, host, readme_scenarios, service

pytestmark = pytest.mark.gpu
ZK_GETDATA = 4


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def host_snapshot(nodes):
    from registrar_b200.batch import Snapshot
    return Snapshot.from_nodes(nodes)


def raw_to_dict(ctx, out):
    """a CAnswers with device arrays, copied out"""
    nq, m = int(out.n_queries), int(out.m)
    return dict(q_kind=_dev(ctx, out.q_kind, nq, np.uint8), q_node=_dev(ctx, out.q_node, nq, np.uint64),
                sec_off=_dev(ctx, out.sec_off, 2 * nq + 1, np.uint64), text=_dev(ctx, out.text, int(out.text_total), np.uint8),
                node_cls=_dev(ctx, out.node_cls, m, np.uint8), unresolved=_dev(ctx, out.unresolved, int(out.n_unresolved), np.uint64),
                n_answers=int(out.n_answers), n_additional=int(out.n_additional))


def compare(got, want):
    """got: an Answers or raw_to_dict's dict; want: rv.resolve's result"""
    g = got if isinstance(got, dict) else dict(q_kind=got.q_kind, q_node=got.q_node, sec_off=got.sec_off, text=got.text,
                                                node_cls=got.node_cls, unresolved=got.unresolved, n_answers=got.n_answers,
                                                n_additional=got.n_additional)
    assert g["node_cls"].tolist() == want["node_cls"]
    assert g["unresolved"].tolist() == want["unresolved"]
    assert g["q_kind"].tolist() == want["q_kind"]
    assert g["q_node"].tolist() == want["q_node"]
    lens = [len(x) for a, b in want["sections"] for x in (a, b)]
    off = np.zeros(len(lens) + 1, np.uint64)
    np.cumsum(lens, out=off[1:])
    assert np.array_equal(g["sec_off"], off)
    assert g["text"].tobytes() == b"".join(a + b for a, b in want["sections"])
    assert (g["n_answers"], g["n_additional"]) == (want["n_answers"], want["n_additional"])


def every_way(ctx, nodes, dh=30, ds=60):
    """host and device snapshots, host and device outputs, all against the restatement; returns the host Answers"""
    want = rv.resolve(nodes, dh, ds)
    got = ctx.resolve(host_snapshot(nodes), dh, ds)
    compare(got, want)
    assert got.m == len(nodes) and got.launches >= 1
    dsnap = device_snapshot(nodes)
    compare(ctx.resolve(dsnap, dh, ds), want)
    compare(raw_to_dict(ctx, ctx.resolve(dsnap, dh, ds, device=True)), want)
    compare(raw_to_dict(ctx, ctx.resolve(host_snapshot(nodes), dh, ds, device=True)), want)
    return got


def test_readme_scenarios(ctx):
    def get(nodes):
        a = every_way(ctx, nodes)
        return {(int(k), rv.name_of(nodes[int(j)][0])): (a.answer(q), a.additional(q))
                for q, (k, j) in enumerate(zip(a.q_kind, a.q_node))}
    check_readme(get)


def random_snapshot(rng, n_dom=12):
    """a mixed registry under /r: directories, services (some without children, one under a service), children of
    every type and class, host records under host records, escaped and non-canonical payloads"""
    types = [b"db_host", b"host", b"load_balancer", b"moray_host", b"ops_host", b"redis_host", b"rr_host", b"databas",
             b"hos\\u0074"]
    nodes = [(b"/r", b"")]

    def addr():
        r = rng.random()
        if r < 0.9:
            return b"10.%d.%d.%d" % (rng.randrange(256), rng.randrange(256), rng.randrange(256))
        return rng.choice([b"10.0.0.256", b"010.1.1.1", b"1.2.3", b"x.y.z.w", b"1.2.3.4\\n"])

    def host_payload():
        typ = rng.choice(types)
        ttl = rng.choice([None, None, 0, 30, 3600, -5, 2 ** 31 - 1])
        ports = rng.choice([None, None, [], [rng.randrange(65536)], [rng.randrange(65536) for _ in range(rng.randrange(1, 5))],
                            [70000]])
        p = host(typ, addr(), ttl, ports)
        r = rng.random()
        if r < 0.04:
            p = p.replace(b'","', b'", "', 1)                  # white space: not canonical
        elif r < 0.06:
            p = host(typ, addr(), ttl, ports, key=b"other")
        elif r < 0.08:
            p = p[:-1]
        return p

    for d in range(n_dom):
        dpath = b"/r/d%d" % d
        kind = rng.random()
        if kind < 0.6:
            nodes.append((dpath, service(rng.choice([b"_http", b"_redis", b"_x-y", b"_a b"]), b"_tcp",
                                         rng.choice([80, 6379, 65535, 65536, 0]), rng.choice([None, 60, 5, -1]))))
        elif kind < 0.8:
            nodes.append((dpath, b""))
        else:
            nodes.append((dpath, host_payload()))
        for k in range(rng.randrange(0, 9)):
            hpath = dpath + b"/h%d" % k
            nodes.append((hpath, host_payload()))
            if rng.random() < 0.15:                                # a host record under a host record
                nodes.append((hpath + b"/z", host_payload()))
        if rng.random() < 0.2:                                     # a service under a service, with a child
            nodes.append((dpath + b"/sub", service(b"_s", b"_udp", 53, None)))
            nodes.append((dpath + b"/sub/c", host(b"rr_host", b"10.9.9.9", None, [1, 2])))
    rng.shuffle(nodes)
    return nodes


@pytest.mark.parametrize("seed", range(6))
def test_random_mixed_snapshots(ctx, seed):
    rng = random.Random(seed)
    nodes = random_snapshot(rng, n_dom=4 + 8 * seed)
    a = every_way(ctx, nodes, dh=rng.choice([0, 30]), ds=rng.choice([60, 2 ** 31 - 1]))
    assert set(a.node_cls.tolist()) <= set(range(8))


def test_every_class_and_empty_snapshot(ctx):
    nodes = random_snapshot(random.Random(99), n_dom=400)
    got = every_way(ctx, nodes)
    assert set(got.node_cls.tolist()) == set(range(8))
    assert {1, 2, 3} <= set(got.q_kind.tolist())
    empty = ctx.resolve(host_snapshot([]), 30, 60)
    assert (empty.m, empty.n_queries, empty.text_total, empty.sec_off.tolist()) == (0, 0, 0, [0])
    only_dirs = every_way(ctx, [(b"/a", b""), (b"/a/b", b"")])
    assert only_dirs.n_queries == 0 and only_dirs.n_unresolved == 0


def test_many_ports_and_large_service(ctx):
    nodes = [(b"/big", service(b"_h", b"_tcp", 8080, 30))]
    nodes += [(b"/big/i%05d" % i, host(b"redis_host", b"10.0.%d.%d" % (i // 256 % 256, i % 256), [None, 10, 90][i % 3],
                                       [None, [], list(range(1, 1 + i % 7))][i % 3])) for i in range(20000)]
    every_way(ctx, nodes)


def test_refusals(ctx):
    from registrar_b200 import _native
    from registrar_b200.batch import Snapshot
    import torch
    nodes = [(b"/a", service()), (b"/a/h", host(b"rr_host")), (b"/b", b""), (b"/a/h", host())]
    for snap in (host_snapshot(nodes), device_snapshot(nodes)):
        with pytest.raises(_native.RegkError, match="node 3 has the path of an earlier node"):
            ctx.resolve(snap, 30, 60)
    good = nodes[:3]
    for dh, ds in ((-1, 60), (30, -1)):
        with pytest.raises(_native.RegkError, match="default TTLs"):
            ctx.resolve(host_snapshot(good), dh, ds)
    cin, keep = host_snapshot(good).cdecode_in()
    o = _native.CResolveOpts(0, 30, 60, 1)
    out = _native.CAnswers()
    assert ctx._lib.regk_resolve(ctx._h, _native.C.byref(cin), _native.C.byref(o), _native.C.byref(out)) == _native.REGK_ERR_INVALID_ARG
    assert "reserved" in ctx._err()
    o = _native.CResolveOpts(0, 30, 60, 0)
    cin.flags |= _native.FLAG_DECODE_LAST
    assert ctx._lib.regk_resolve(ctx._h, _native.C.byref(cin), _native.C.byref(o), _native.C.byref(out)) == _native.REGK_ERR_INVALID_ARG
    d = device_snapshot(good)
    bad = d.json_off.clone()
    bad[2] = bad[3] + 5                                            # node 1 ends before it starts
    with pytest.raises(_native.RegkError, match="at node 1"):
        ctx.resolve(Snapshot(d.path_bytes, d.path_off, d.json_bytes, bad), 30, 60)
    bad = d.path_off.clone()
    bad[3] = d.path_bytes.numel() + 1                              # node 2 reaches past the total
    with pytest.raises(_native.RegkError, match="at node 2"):
        ctx.resolve(Snapshot(d.path_bytes, bad, d.json_bytes, d.json_off), 30, 60)
    compare(ctx.resolve(d, 30, 60), rv.resolve(good, 30, 60))     # the context is still usable


def test_pipeline_from_read_replies(ctx):
    """compose a fleet batch, frame its getData, answer it, read the replies on the GPU and resolve the snapshot as it
    stands: the batch's own host records only, so its HOST_A answers"""
    from registrar_b200 import synth
    b = synth.generate("config2", n=20000)
    got = ctx.register_batch(b)
    paths = [got.path(i) for i in range(got.n)]
    fb, fo, _ = ctx.jute_requests(ZK_GETDATA, xid_base=11)
    assert fb.tobytes() == ru.getdata_frames(paths, 11)
    n = got.n
    stream = ru.device_replies(got.json_bytes, got.json_off.astype(np.uint64), 11, np.zeros(n, np.int32), np.zeros(n, np.int64),
                               missing=np.arange(n) % 17 == 3)
    rep = ctx.read_replies(stream)
    assert rep.n_found == n - len(range(3, n, 17))
    nodes = [(paths[k], got.json(k)) for k in rep.node_rec.tolist()]
    want = rv.resolve(nodes, 30, 60)
    a = ctx.resolve(rep, 30, 60)
    compare(a, want)
    assert a.n_queries == sum(1 for k in want["q_kind"] if k == rv.HOST_A) > 0


def fleet_nodes(n, ndom=1000, seed=3):
    """n config 2 host records collapsed onto `ndom` domains, plus one service record per domain"""
    from registrar_b200 import _native, synth
    rng = np.random.default_rng(seed)
    b = synth.generate("config2", n=n)
    idx = rng.integers(0, ndom, n)
    lens = np.diff(b.domain_off)[idx]
    off = np.zeros(n + 1, np.uint32)
    np.cumsum(lens, out=off[1:])
    pos = np.repeat(b.domain_off[:-1][idx].astype(np.int64) - off[:-1].astype(np.int64), lens) + np.arange(int(off[-1]))
    b.domain_bytes = b.domain_bytes[pos]
    b.domain_off = off
    c = _native.Context(0)
    try:
        got = c.register_batch(b)
    finally:
        c.close()
    return got, idx


def fleet_snapshot(got, idx, ndom, seed=5):
    """the records' nodes followed by one service record per domain (port, ttl varied): (path/json arrays, nodes)"""
    rng = random.Random(seed)
    po, jo = got.path_off.astype(np.int64), got.json_off.astype(np.int64)
    first = {}
    for i, d in enumerate(idx[:200000].tolist()):
        first.setdefault(d, i)
    svc = []
    for d in sorted(first):
        i = first[d]
        p = got.path_bytes[po[i]:po[i + 1]].tobytes()
        svc.append((p[:p.rfind(b"/")], service(b"_http", b"_tcp", rng.choice([80, 443, 8080]), rng.choice([None, 60]))))
    pb = np.concatenate([got.path_bytes[:po[-1]], np.frombuffer(b"".join(p for p, _ in svc), np.uint8)])
    jb = np.concatenate([got.json_bytes[:jo[-1]], np.frombuffer(b"".join(j for _, j in svc), np.uint8)])
    po2 = np.concatenate([po, po[-1] + np.cumsum([len(p) for p, _ in svc])]).astype(np.uint64)
    jo2 = np.concatenate([jo, jo[-1] + np.cumsum([len(j) for _, j in svc])]).astype(np.uint64)
    return pb, po2, jb, jo2


@pytest.mark.slow
def test_fleet_million_hosts_under_a_thousand_services(ctx):
    import torch
    from registrar_b200.batch import Snapshot
    got, idx = fleet_nodes(1_000_000)
    pb, po, jb, jo = fleet_snapshot(got, idx, 1000)
    m = len(po) - 1
    assert m == 1_000_000 + 1000
    pbs, jbs = pb.tobytes(), jb.tobytes()
    nodes = [(pbs[po[j]:po[j + 1]], jbs[jo[j]:jo[j + 1]]) for j in range(m)]
    want = rv.resolve(nodes, 30, 60)
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()
    a = ctx.resolve(Snapshot(t(pb, np.uint8), t(po, np.int64), t(jb, np.uint8), t(jo, np.int64)), 30, 60)
    compare(a, want)
    n_srv = sum(1 for k in want["q_kind"] if k == rv.SERVICE_SRV)
    assert n_srv == 1000 and a.n_additional > 500_000
