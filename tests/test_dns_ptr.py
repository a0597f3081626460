"""regk_dns_answer with REGK_DNS_PTR on the GPU, bit for bit against the restatement in dns_ptr_util through host and
device input and output: the README scenarios and random snapshots with addresses shared by aliases, queryable
service children and non-queryable children, reverse-name query mixes (partial, leading zero, 256, upper case,
absent, 0.0.0.0 and 255.255.255.255), flag-off parity, truncation of one address shared by 2 000 long names, the
reverse index's launch counts, PTR answers after a watched walk's refresh, and a 4 M host fleet."""
import random

import numpy as np
import pytest

import dns_ptr_util as pu
import dns_util as du
import resolve_util as rv
from test_dns import case_mix, compare, host_dict, host_snapshot, random_queries, raw
from test_dns_cpu import zone_queries
from test_reconcile import device_snapshot
from test_resolve import fleet_nodes, fleet_snapshot, random_snapshot
from test_resolve_cpu import host, readme_scenarios, service

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def every_way(ctx, zone, msgs, udp=1232, tcp=False):
    """with the flag: host and device messages, host and device outputs, against the restatement; without it: every
    non-reverse message's bytes unchanged, and the whole output dns_util's"""
    import torch
    want = pu.answer_all(zone, msgs, udp, tcp)
    mb, mo = du.pack(msgs)
    r = ctx.answer_dns(mb, mo, udp, tcp, ptr=True)
    compare(host_dict(r), want, msgs)
    dm, do = torch.from_numpy(mb).cuda(), torch.from_numpy(mo).cuda()
    compare(host_dict(ctx.answer_dns(dm, do, udp, tcp, ptr=True)), want, msgs)
    compare(raw(ctx, ctx.answer_dns(dm, do, udp, tcp, device=True, ptr=True)), want, msgs)
    compare(raw(ctx, ctx.answer_dns(mb, mo, udp, tcp, device=True, ptr=True)), want, msgs)
    off = ctx.answer_dns(mb, mo, udp, tcp)
    compare(host_dict(off), du.answer_all(zone, msgs, udp, tcp), msgs)
    for i, m in enumerate(msgs):
        if pu.reverse_addr(du.parse(m)["labels"]) is None:
            assert off.response(i) == r.response(i) and off.status[i] == r.status[i], i
    return r


def reverse_queries(rng, addrs, n):
    """PTR / A / SRV / ANY on reverse names of `addrs` and of absent addresses, in every form the rules name"""
    out = []
    for _ in range(n):
        a = rng.choice(addrs) if addrs and rng.random() < 0.7 else b"%d.%d.%d.%d" % tuple(rng.randrange(256) for _ in range(4))
        o = a.split(b".")
        r = rng.random()
        if r < 0.55:
            name = pu.reverse_name(a)
        elif r < 0.65:
            name = case_mix(rng, pu.reverse_name(a).upper())
        elif r < 0.72:
            name = b".".join(reversed(o[rng.randrange(1, 4):])) + b".in-addr.arpa"            # partial
        elif r < 0.79:
            k = rng.randrange(4)
            o[k] = b"0" + o[k]                                                              # leading zero
            name = pu.reverse_name(b".".join(o))
        elif r < 0.86:
            o[rng.randrange(4)] = rng.choice([b"256", b"999", b"1000", b"x"])
            name = pu.reverse_name(b".".join(o))
        elif r < 0.93:
            name = pu.reverse_name(a) + rng.choice([b".x", b"x"])
        else:
            name = rng.choice([b"in-addr.arpa", b"arpa", b"0.0.0.0.in-addr.arpa", b"255.255.255.255.in-addr.arpa"])
        opt = rng.choice([None, None, (rng.choice([0, 512, 1232, 4096]), 0, rng.randrange(2)), (1232, 1, 0)])
        out.append(du.query(name, rng.choice([pu.T_PTR] * 4 + [du.T_A, du.T_SRV, du.T_ANY]), ident=rng.randrange(65536),
                            rd=rng.randrange(2), qclass=rng.choice([1] * 6 + [3]), opt=opt))
    return out


def addrs_of(zone):
    return sorted(pu.reverse_map(zone))


def test_readme_scenarios(ctx):
    rng = random.Random(0)
    for nodes in readme_scenarios().values():
        ctx.resolve(host_snapshot(nodes), 30, 60)
        zone = du.Zone(nodes)
        msgs = zone_queries(zone, nodes, rng) + reverse_queries(rng, addrs_of(zone), 300)
        r = every_way(ctx, zone, msgs)
        assert r.n_status[du.ANSWER] > 0


def shared_snapshot(rng, n_dom):
    """random_snapshot with addresses deliberately shared: aliases of hosts, queryable service children and
    non-queryable children at one address, and hosts at 0.0.0.0 and 255.255.255.255"""
    nodes = random_snapshot(rng, n_dom=n_dom)
    pool = [b"10.0.0.1", b"10.0.0.2", b"0.0.0.0", b"255.255.255.255", b"172.27.10.72"]
    extra = [(b"/s", service(b"_http", b"_tcp", 80, 60))]
    for i in range(60):
        a = rng.choice(pool)
        typ = rng.choice([b"host", b"load_balancer", b"redis_host", b"ops_host", b"rr_host", b"moray_host", b"db_host"])
        parent = rng.choice([b"/s", b"/a"])
        extra.append((parent + b"/h%d" % i, host(typ, a, rng.choice([None, 0, 7, 300]), rng.choice([None, [80], []]))))
    extra.append((b"/a", b""))
    extra += [(b"/bad/h%d" % i, host(b"host", pool[i % len(pool)], -1)) for i in range(3)]
    extra.append((b"/arpa/in-addr/10/0/0/1", host(b"host", b"10.0.0.1")))          # a reverse name that owns A too
    nodes += extra
    rng.shuffle(nodes)
    return nodes


@pytest.mark.parametrize("seed", range(4))
def test_random_snapshots_and_queries(ctx, seed):
    rng = random.Random(seed)
    nodes = shared_snapshot(rng, 6 + 8 * seed)
    dh, ds = rng.choice([0, 30]), rng.choice([60, 2 ** 31 - 1])
    snap = device_snapshot(nodes) if seed % 2 else host_snapshot(nodes)
    ctx.resolve(snap, dh, ds)
    zone = du.Zone(nodes, dh, ds)
    msgs = random_queries(rng, nodes, zone, 1500) + reverse_queries(rng, addrs_of(zone), 2500)
    rng.shuffle(msgs)
    for udp, tcp in ((512, False), (1232, False), (65535, True)):
        r = every_way(ctx, zone, msgs, udp, tcp)
    assert r.n_status[du.ANSWER] and r.n_status[du.NODATA] and r.n_status[du.NXDOMAIN]
    ptr_answers = [i for i, m in enumerate(msgs) if r.status[i] == du.ANSWER and du.parse(m)["qtype"] == pu.T_PTR]
    assert len(ptr_answers) > 100


def test_truncation_of_a_shared_address(ctx):
    a = b"10.20.30.40"
    label = b"i" * 50
    nodes = [(b"/us/example/%s%04d" % (label, i), host(b"host", a, i % 3 or None)) for i in range(2000)]
    ctx.resolve(host_snapshot(nodes), 30, 60)
    zone = du.Zone(nodes)
    name = pu.reverse_name(a)
    rr = 14 + len(rv.name_of(nodes[0][0]))
    msgs = [du.query(name, pu.T_PTR)] + [du.query(name, pu.T_PTR, opt=(s, 0, 1)) for s in (511, 512, 513, 1232, 4096, 65535)]
    for udp, tcp in ((512, False), (1232, False), (4096, False), (65535, False), (1232, True)):
        r = every_way(ctx, zone, msgs, udp, tcp)
        for i, m in enumerate(msgs):
            qend = len(du.query(name, pu.T_PTR))
            resp = r.response(i)
            body = len(resp) - qend - (11 if i else 0)
            assert body % rr == 0 and body // rr == int.from_bytes(resp[6:8], "big")
            assert r.tc[i] == (body // rr < 2000) == bool(resp[2] & 2)


def test_index_launch_counts(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    try:
        nodes = readme_scenarios()["plain"] + [(b"/us/x", service()), (b"/us/x/h", host(b"redis_host", b"10.0.0.5"))]
        msgs = [du.query(pu.reverse_name(b"172.27.10.72"), pu.T_PTR), du.query(b"h.x.us"),
                du.query(b"_http._tcp.x.us", du.T_SRV)]
        mb, mo = du.pack(msgs)
        zone = du.Zone(nodes)
        c.resolve(host_snapshot(nodes), 30, 60)
        first = c.answer_dns(mb, mo, ptr=True)                  # preparation (2) and the index (2 + sort + 2)
        plain = c.answer_dns(mb, mo)                            # neither builds nor drops the index
        again = c.answer_dns(mb, mo, ptr=True)
        assert first.launches == again.launches + 2 + 5
        assert host_dict(again) == pu.answer_all(zone, msgs) and host_dict(plain) == du.answer_all(zone, msgs)
        c.resolve(host_snapshot(nodes), 30, 60)                 # a new resolve: the index is rebuilt
        plain2 = c.answer_dns(mb, mo)
        assert plain2.launches == plain.launches + 2
        rebuilt = c.answer_dns(mb, mo, ptr=True)
        assert rebuilt.launches == again.launches + 5
        assert c.answer_dns(mb, mo, ptr=True).launches == again.launches
        assert host_dict(rebuilt) == pu.answer_all(zone, msgs)
        empty = [(b"/us/x", service())]                         # no host node: the compaction alone
        c.resolve(host_snapshot(empty), 30, 60)
        r = c.answer_dns(mb, mo, ptr=True)
        assert host_dict(r) == pu.answer_all(du.Zone(empty), msgs) and r.n_status[du.NXDOMAIN] == 2
    finally:
        c.close()


def test_answers_follow_a_watched_walk(built):
    import walk_watch_util as ww
    from registrar_b200 import _native
    c = _native.Context(0)
    session = 7
    try:
        zk = ww.WalkZooKeeper()
        zk.create(b"/r", b"", 0, False)
        for s in range(3):
            zk.create(b"/r/s%d" % s, service(b"_http", b"_tcp", 80, 60), 0, False)
            for i in range(30):
                zk.create(b"/r/s%d/i%d" % (s, i), host(b"redis_host", b"10.1.0.%d" % (i % 7), None, [6379]), 0, False)
        c.walk([b"/r"], lambda fb: zk.serve(fb, session), watch=True)

        def check():
            c.walk_resolve(30, 60)
            snap = c._walk.snapshot()
            pb, po, jb, jo = snap.path_bytes.tobytes(), snap.path_off, snap.json_bytes.tobytes(), snap.json_off
            nodes = [(pb[po[j]:po[j + 1]], jb[jo[j]:jo[j + 1]]) for j in range(len(po) - 1)]
            zone = du.Zone(nodes)
            addrs = [b"10.1.0.%d" % k for k in range(10)] + [b"10.9.9.%d" % k for k in range(3)]
            msgs = [du.query(pu.reverse_name(a), t) for a in addrs for t in (pu.T_PTR, du.T_A)]
            msgs += [du.query(rv.name_of(p)) for p, _ in nodes]
            every_way(c, zone, msgs)
            return zone

        check()
        rng = random.Random(1)
        for rnd in range(3):
            for i in rng.sample(range(30), 6):                  # readdressed
                p = b"/r/s%d/i%d" % (rnd, i)
                if p in zk.nodes:
                    zk.set_data(p, host(b"redis_host", b"10.1.0.%d" % rng.randrange(10), None, [6379]))
            zk.delete(b"/r/s%d/i%d" % ((rnd + 1) % 3, rnd))    # deleted
            zk.create(b"/r/s%d/new%d" % (rnd, rnd), host(b"host", b"10.9.9.%d" % rnd), 0, False)   # created
            c.walk_events(np.frombuffer(zk.take_events(session), np.uint8))
            c.refresh_walk(lambda fb: zk.serve(fb, session))
            mb, mo = du.pack([du.query(b"1.0.1.10.in-addr.arpa", pu.T_PTR)])
            with pytest.raises(RuntimeError, match="resolve it again"):
                c.answer_dns(mb, mo, ptr=True)
            zone = check()
            assert pu.reverse_map(zone)[b"10.9.9.%d" % rnd][-1][2] == b"new%d.s%d.r" % (rnd, rnd)
    finally:
        c.close()


@pytest.mark.slow
def test_fleet_four_million_hosts(ctx):
    """10 M device-resident queries, 20 % PTR, against 4 M config 2 records under 1 000 service records; every count
    checked against the restatement of the query pool, a sample of 50 000 responses byte for byte"""
    import re
    import torch
    from registrar_b200.batch import Snapshot
    n = 4_000_000
    got, idx = fleet_nodes(n)
    pb, po, jb, jo = fleet_snapshot(got, idx, 1000)
    m = len(po) - 1
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()
    snap = Snapshot(t(pb, np.uint8), t(po, np.int64), t(jb, np.uint8), t(jo, np.int64))
    ctx.resolve(snap, 30, 60)
    # the restatement over the nodes the query pool can reach: the sampled hosts, every node at a sampled address
    rng = random.Random(11)
    jbs, pbs = jb.tobytes(), pb.tobytes()

    def addr(j):
        d = jbs[jo[j]:jo[j + 1]]
        k = d.find(b'"address":"') + 11
        return d[k:d.index(b'"', k)]
    addr_of = {}
    for j in range(n):
        addr_of.setdefault(addr(j), []).append(j)
    sample = rng.sample(range(n), 2000)
    want_addrs = sorted({addr(j) for j in sample})
    keep = sorted({j for a in want_addrs for j in addr_of[a]} | set(sample))
    sub = [(pbs[po[j]:po[j + 1]], jbs[jo[j]:jo[j + 1]]) for j in keep]
    zone = du.Zone(sub)
    back = np.array(keep + [du.NONE], np.uint64)
    hosts = [rv.name_of(pbs[po[j]:po[j + 1]]) for j in sample]
    pool = ([du.query(case_mix(rng, h)) for h in hosts] + [du.query(h, du.T_AAAA) for h in hosts[:500]] +
            [du.query(b"nx.example")])
    n_fwd = len(pool)
    pool += [du.query(pu.reverse_name(a), pu.T_PTR, opt=rng.choice([None, (1232, 0, 0)])) for a in want_addrs]
    pool += [du.query(pu.reverse_name(b"192.168.%d.%d" % (k // 256, k % 256)), pu.T_PTR) for k in range(200)]
    pool += [du.query(pu.reverse_name(a), du.T_A) for a in want_addrs[:200]]
    gen = np.random.default_rng(1)
    is_ptr = gen.random(10_000_000) < 0.2
    pick = np.where(is_ptr, gen.integers(n_fwd, len(pool), 10_000_000), gen.integers(0, n_fwd, 10_000_000))
    lens = np.array([len(x) for x in pool], np.int64)
    blob = np.frombuffer(b"".join(pool), np.uint8).copy()
    pstart = np.zeros(len(pool), np.int64)
    np.cumsum(lens[:-1], out=pstart[1:])
    off = np.zeros(len(pick) + 1, np.int64)
    np.cumsum(lens[pick], out=off[1:])
    dblob, dstarts, dpick = torch.from_numpy(blob).cuda(), torch.from_numpy(pstart).cuda(), torch.from_numpy(pick).cuda()
    doff = torch.from_numpy(off).cuda()
    bpos = torch.arange(int(off[-1]), device="cuda", dtype=torch.int64)
    which = torch.searchsorted(doff[1:], bpos, right=True)
    msgs = dblob[dstarts[dpick[which]] + bpos - doff[which]]
    del bpos, which
    r = ctx.answer_dns(msgs, doff, 1232, ptr=True)
    assert r.k == 10_000_000 and sum(r.n_status) == r.k
    rmap = pu.reverse_map(zone)
    want = [pu.answer(zone, x, 1232, rmap=rmap) for x in pool]
    want = [(s, tc, int(back[node]) if node != du.NONE else du.NONE, b) for s, tc, node, b in want]
    wl = np.array([len(w[3]) for w in want], np.int64)
    assert np.array_equal(np.diff(r.resp_off.astype(np.int64)), wl[pick])
    ws = np.array([w[0] for w in want])
    assert r.n_status == np.bincount(ws[pick], minlength=8).tolist()
    assert r.n_truncated == int(np.array([w[1] for w in want])[pick].sum())
    assert (r.status[is_ptr] == du.ANSWER).sum() > 1_000_000
    for i in np.random.default_rng(2).integers(0, len(pick), 50_000).tolist():
        w = want[pick[i]]
        assert (r.status[i], r.tc[i], r.node[i], r.response(i)) == (w[0], w[1], w[2], w[3])
