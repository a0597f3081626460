"""regk_dns_answer on the GPU, bit for bit against the restatement in dns_util: the README scenarios, random mixed
snapshots with random query mixes (0x20 case, A / SRV / AAAA / ANY, names that own nothing, bad label bytes, every
node class, malformed messages), truncation at the edges of every size limit, host and device input and output, the
state rules, the refusals, a cross-check of every regk_resolve query over TCP with dnspython, and 10 M queries."""
import random

import numpy as np
import pytest

import dns_util as du
import resolve_util as rv
from test_dns_cpu import decoded, mutations, rrsets, zone_queries
from test_reconcile import _dev, device_snapshot
from test_resolve import fleet_nodes, fleet_snapshot, random_snapshot
from test_resolve_cpu import host, readme_scenarios, service

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def host_snapshot(nodes):
    from registrar_b200.batch import Snapshot
    return Snapshot.from_nodes(nodes)


def raw(ctx, out):
    k, total = int(out.k), int(out.resp_total)
    return dict(resp_off=_dev(ctx, out.resp_off, k + 1, np.uint64).tolist(), resp=_dev(ctx, out.resp, total, np.uint8).tobytes(),
                status=_dev(ctx, out.status, k, np.uint8).tolist(), tc=_dev(ctx, out.tc, k, np.uint8).tolist(),
                node=_dev(ctx, out.node, k, np.uint64).tolist(), n_status=list(out.n_status), n_truncated=int(out.n_truncated))


def host_dict(r):
    return dict(resp_off=r.resp_off.tolist(), resp=r.resp.tobytes(), status=r.status.tolist(), tc=r.tc.tolist(),
                node=r.node.tolist(), n_status=r.n_status, n_truncated=r.n_truncated)


def compare(got, want, msgs):
    for i in range(len(msgs)):
        g = got["resp"][got["resp_off"][i]:got["resp_off"][i + 1]]
        w = want["resp"][want["resp_off"][i]:want["resp_off"][i + 1]]
        assert (got["status"][i], got["tc"][i], got["node"][i], g) == (want["status"][i], want["tc"][i], want["node"][i], w), \
            (i, msgs[i].hex())
    assert got == want


def every_way(ctx, zone, msgs, udp=1232, tcp=False):
    """host and device messages, host and device outputs, against the restatement (the last resolve is zone's)"""
    import torch
    want = du.answer_all(zone, msgs, udp, tcp)
    mb, mo = du.pack(msgs)
    r = ctx.answer_dns(mb, mo, udp, tcp)
    compare(host_dict(r), want, msgs)
    dm, do = torch.from_numpy(mb).cuda(), torch.from_numpy(mo).cuda()
    compare(host_dict(ctx.answer_dns(dm, do, udp, tcp)), want, msgs)
    compare(raw(ctx, ctx.answer_dns(dm, do, udp, tcp, device=True)), want, msgs)
    compare(raw(ctx, ctx.answer_dns(mb, mo, udp, tcp, device=True)), want, msgs)
    return r


def case_mix(rng, name):
    return bytes(c ^ 0x20 if chr(c).isalpha() and rng.random() < 0.5 else c for c in name)


def random_queries(rng, nodes, zone, n):
    names = [rv.name_of(p) for p, _ in nodes]
    srv = [zone.rec[j][1] + b"." + zone.rec[j][2] + b"." + rv.name_of(nodes[j][0]) for j in zone.srv]
    bad = mutations()
    out = []
    for _ in range(n):
        r = rng.random()
        opt = rng.choice([None, None, (rng.choice([0, 511, 512, 900, 1232, 1500, 4096, 65535]), 0, rng.randrange(2)),
                          (1232, 1, 0)])
        if r < 0.4 and names:
            nm = case_mix(rng, rng.choice(names))
        elif r < 0.7 and srv:
            nm = case_mix(rng, rng.choice(srv))
        elif r < 0.8:
            nm = rng.choice([b"nx.r", b"d1.r.x", b"a*b.d1.r", b"_http._tcp", b"", b"h0.d0.r.extra"])
        else:
            out.append(rng.choice(bad))
            continue
        out.append(du.query(nm, rng.choice([du.T_A, du.T_A, du.T_SRV, du.T_SRV, du.T_AAAA, du.T_ANY]), ident=rng.randrange(65536),
                            rd=rng.randrange(2), qclass=rng.choice([1, 1, 1, 1, 3, 255]), opt=opt))
    return out


def test_readme_scenarios(ctx):
    rng = random.Random(0)
    for nodes in readme_scenarios().values():
        ctx.resolve(host_snapshot(nodes), 30, 60)
        zone = du.Zone(nodes)
        msgs = zone_queries(zone, nodes, rng)
        r = every_way(ctx, zone, msgs)
        assert r.n_status[du.ANSWER] > 0


@pytest.mark.parametrize("seed", range(5))
def test_random_snapshots_and_queries(ctx, seed):
    rng = random.Random(seed)
    nodes = random_snapshot(rng, n_dom=6 + 10 * seed)
    if seed % 2:
        nodes = [(p.replace(b"/d1", b"/D1"), d) for p, d in nodes]            # a path no name reaches
    dh, ds = rng.choice([0, 30]), rng.choice([60, 2 ** 31 - 1])
    snap = device_snapshot(nodes) if seed % 2 else host_snapshot(nodes)   # kept alive: answers read its paths
    ctx.resolve(snap, dh, ds)
    zone = du.Zone(nodes, dh, ds)
    msgs = random_queries(rng, nodes, zone, 3000)
    for udp, tcp in ((512, False), (1232, False), (4096, False), (65535, True)):
        r = every_way(ctx, zone, msgs, udp, tcp)
    assert sum(r.n_status) == len(msgs)
    assert all(r.n_status[s] for s in (du.ANSWER, du.NODATA, du.NXDOMAIN, du.FORMERR, du.REFUSED, du.BADVERS, du.DROPPED))


def edge_service(svc_name, target, qend, opt):
    """a service whose SRV answers alone make a response of exactly `target` bytes; children with ports [],
    several ports and the service's port; returns the nodes"""
    path = b"/" + b"/".join(reversed(svc_name.split(b".")))
    nodes = [(path, service(b"_e", b"_tcp", 7000, 60))]
    rest = target - qend - (11 if opt else 0)
    i = 0
    while rest > 0:
        lab = b"c%04d" % i
        lc = len(lab) + 1 + len(svc_name)
        ports = [None, [], [1, 2, 3], [9]][i % 4]
        need = (1 if ports is None else len(ports)) * (20 + lc)
        small = 20 + len(svc_name) + 3                                   # the smallest child that can follow
        if rest != need and rest - need < small:
            ports, need = [5], 20 + lc
            if rest != need and rest - need < small:
                lab = b"c" * (rest - 21 - len(svc_name))             # the last child makes it exact
                assert 1 <= len(lab) <= 63, rest
                need = rest
        nodes.append((path + b"/" + lab, host(b"rr_host", b"10.1.%d.%d" % (i // 250, i % 250), None, ports)))
        rest -= need
        i += 1
    return nodes


@pytest.mark.parametrize("limit,udp,tcp,osize", [(512, 1232, False, None), (900, 1232, False, 900),
                                                  (1232, 1232, False, 4096), (65535, 1232, True, 1232)])
def test_truncation_edges(ctx, limit, udp, tcp, osize):
    svc = b"edge.example.us"
    q = b"_e._tcp." + svc
    opt = None if osize is None else (osize, 0, 1)
    qend = len(du.query(q, du.T_SRV))
    for d in (-1, 0, 1):
        nodes = edge_service(svc, limit + d, qend, opt is not None)
        ctx.resolve(host_snapshot(nodes), 30, 60)
        zone = du.Zone(nodes)
        msgs = [du.query(q, du.T_SRV, opt=opt), du.query(svc, du.T_A, opt=opt), du.query(b"c0000." + svc, du.T_A, opt=opt)]
        r = every_way(ctx, zone, msgs, udp, tcp)
        assert r.tc[0] == (d > 0) and len(r.response(0)) <= limit
        if d <= 0:
            assert len(r.response(0)) == limit + d


def test_state_rules(ctx, built):
    from registrar_b200 import _native
    fresh = _native.Context(0)
    try:
        mb, mo = du.pack([du.query(b"x.us")])
        with pytest.raises(_native.RegkError, match="no successful regk_resolve") as e:
            fresh.answer_dns(mb, mo)
        assert e.value.code == _native.REGK_ERR_STATE
        a = [(b"/us/a", service()), (b"/us/a/h", host(b"rr_host", b"10.0.0.1"))]
        b = [(b"/us/b", host(b"host", b"10.0.0.2"))]
        fresh.resolve(host_snapshot(a), 30, 60)
        msgs = [du.query(b"a.us"), du.query(b"b.us"), du.query(b"_http._tcp.a.us", du.T_SRV)]
        mb, mo = du.pack(msgs)
        first = fresh.answer_dns(mb, mo)
        second = fresh.answer_dns(mb, mo)
        assert first.launches == second.launches + 2                       # the preparation ran once
        assert first.status.tolist() == [du.ANSWER, du.NXDOMAIN, du.ANSWER]
        assert host_dict(second) == du.answer_all(du.Zone(a), msgs)
        fresh.resolve(host_snapshot(b), 30, 60)                            # a second resolve replaces the first
        third = fresh.answer_dns(mb, mo)
        assert third.launches == first.launches
        assert host_dict(third) == du.answer_all(du.Zone(b), msgs)
        with pytest.raises(_native.RegkError):
            fresh.resolve(host_snapshot(b + b), 30, 60)                    # a failed resolve: nothing to answer from
        with pytest.raises(_native.RegkError, match="no successful regk_resolve"):
            fresh.answer_dns(mb, mo)
    finally:
        fresh.close()


def test_refusals(ctx):
    import torch
    from registrar_b200 import _native
    nodes = [(b"/us/a", service()), (b"/us/a/h", host(b"rr_host", b"10.0.0.1"))]
    ctx.resolve(host_snapshot(nodes), 30, 60)
    msgs = [du.query(b"a.us")] * 4
    mb, mo = du.pack(msgs)
    L, C = ctx._lib, _native.C

    def call(cin, opts):
        out = _native.CDnsOut()
        return L.regk_dns_answer(ctx._h, C.byref(cin), C.byref(opts), C.byref(out))

    cin = lambda o=mo, flags=0, res=0: _native.CDnsIn(mb.ctypes.data, o.ctypes.data, len(o) - 1, int(o[-1]), flags, res)
    ok = _native.CDnsOpts(0, 1232)
    assert call(cin(), ok) == 0
    for c, o, text in ((cin(res=1), ok, "reserved"), (cin(flags=4), ok, "unknown input flag"),
                       (cin(), _native.CDnsOpts(1 << 9, 1232), "unknown flag"), (cin(), _native.CDnsOpts(0, 511), "udp_payload 511"),
                       (cin(), _native.CDnsOpts(0, 65536), "udp_payload 65536")):
        assert call(c, o) == _native.REGK_ERR_INVALID_ARG and text in ctx._err()
    assert L.regk_dns_answer(ctx._h, None, C.byref(ok), C.byref(_native.CDnsOut())) == _native.REGK_ERR_INVALID_ARG
    cases = ((1, lambda o: o.__setitem__(2, o[1] - 1), True), (3, lambda o: o.__setitem__(4, o[4] + 1), False),
             (2, lambda o: o.__setitem__(3, o[2] + 70000), True))
    dm = torch.from_numpy(mb).cuda()
    for bad_at, fix, on_host in cases:                                 # a host total is off[k] by definition
        o = mo.copy()
        fix(o)
        if on_host:
            with pytest.raises(_native.RegkError, match="message %d:" % bad_at):
                ctx.answer_dns(mb, o)
        with pytest.raises(_native.RegkError, match="message %d:" % bad_at):
            ctx.answer_dns(dm, torch.from_numpy(o).cuda())
    long_msg = du.query(b"a.us") + b"\0" * 65530
    lb, lo = du.pack([du.query(b"a.us"), long_msg])
    with pytest.raises(_native.RegkError, match="message 1:"):
        ctx.answer_dns(lb, lo)
    with pytest.raises(_native.RegkError, match="message 1:"):
        ctx.answer_dns(torch.from_numpy(lb).cuda(), torch.from_numpy(lo).cuda())
    do = torch.zeros(len(mo) + 1, dtype=torch.int64, device="cuda")
    do[1:] = torch.from_numpy(mo).cuda()
    cm = _native.CDnsIn(dm.data_ptr(), do.data_ptr() + 4, len(mo) - 1, int(mo[-1]), _native.FLAG_IN_DEVICE, 0)
    assert call(cm, ok) == _native.REGK_ERR_INVALID_ARG and "misaligned" in ctx._err()
    r = ctx.answer_dns(mb, mo)                                             # still usable
    assert r.status.tolist() == [du.ANSWER] * 4


def test_cross_check_every_resolve_query_over_tcp(ctx):
    """each regk_resolve query asked once over TCP decodes, with dnspython, to that query's text sections"""
    pytest.importorskip("dns")
    import dns.message
    nodes = random_snapshot(random.Random(7), n_dom=120)
    nodes += [(b"/us/big", service(b"_h", b"_tcp", 8080, 30))]
    nodes += [(b"/us/big/i%03d" % i, host(b"redis_host", b"10.0.0.%d" % i, [None, 10][i % 2], [None, [], [1, 2]][i % 3]))
              for i in range(200)]
    a = ctx.resolve(host_snapshot(nodes), 30, 60)
    recs = {j: rv.classify(*nodes[j])[1] for j in set(a.q_node.tolist())}
    msgs = []
    for kind, j in zip(a.q_kind.tolist(), a.q_node.tolist()):
        name = rv.name_of(nodes[j][0])
        if name != name.lower():
            msgs.append(None)
            continue
        msgs.append(du.query(recs[j][1] + b"." + recs[j][2] + b"." + name, du.T_SRV) if kind == rv.SERVICE_SRV else du.query(name))
    asked = [m for m in msgs if m is not None]
    r = ctx.answer_dns(*du.pack(asked), tcp=True)
    assert r.n_status[du.ANSWER] == len(asked) and r.n_truncated == 0
    i = 0
    for q, m in enumerate(msgs):
        if m is None:
            continue
        got = dns.message.from_wire(r.response(i))
        assert decoded(got.answer) == rrsets(a.answer(q))
        add = a.additional(q)
        if len(r.response(i)) < 0x3000:
            assert decoded(got.additional) == rrsets(add)
        i += 1
    assert i > 100


@pytest.mark.slow
def test_ten_million_queries(ctx):
    """10 M device-resident queries against a million config 2 records under 1 000 service records; a sample of
    50 000 compared with the restatement, every count checked"""
    import torch
    from registrar_b200.batch import Snapshot
    got, idx = fleet_nodes(1_000_000)
    pb, po, jb, jo = fleet_snapshot(got, idx, 1000)
    m = len(po) - 1
    pbs, jbs = pb.tobytes(), jb.tobytes()
    nodes = [(pbs[po[j]:po[j + 1]], jbs[jo[j]:jo[j + 1]]) for j in range(m)]
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()
    snap = Snapshot(t(pb, np.uint8), t(po, np.int64), t(jb, np.uint8), t(jo, np.int64))
    ctx.resolve(snap, 30, 60)
    zone = du.Zone(nodes)
    rng = random.Random(11)
    hosts = [rv.name_of(nodes[j][0]) for j in rng.sample(range(1_000_000), 2000)]
    svcs = [rv.name_of(nodes[j][0]) for j in range(1_000_000, m)]
    pool = ([du.query(case_mix(rng, h)) for h in hosts] + [du.query(b"_http._tcp." + s, du.T_SRV, opt=(1232, 0, 0)) for s in svcs]
            + [du.query(s) for s in svcs] + [du.query(h, du.T_AAAA) for h in hosts[:500]] + [du.query(b"nx.example")])
    pick = np.random.default_rng(1).integers(0, len(pool), 10_000_000)
    lens = np.array([len(x) for x in pool], np.int64)
    blob = np.frombuffer(b"".join(pool), np.uint8)
    starts = np.zeros(len(pool), np.int64)
    np.cumsum(lens[:-1], out=starts[1:])
    off = np.zeros(len(pick) + 1, np.int64)
    np.cumsum(lens[pick], out=off[1:])
    dblob, dstarts, dpick = torch.from_numpy(blob).cuda(), torch.from_numpy(starts).cuda(), torch.from_numpy(pick).cuda()
    doff = torch.from_numpy(off).cuda()
    pos = torch.arange(int(off[-1]), device="cuda", dtype=torch.int64)
    which = torch.searchsorted(doff[1:], pos, right=True)
    msgs = dblob[dstarts[dpick[which]] + pos - doff[which]]
    del pos, which
    r = ctx.answer_dns(msgs, doff, 1232)
    assert r.k == 10_000_000 and sum(r.n_status) == r.k
    want = [du.answer(zone, x, 1232) for x in pool]
    wl = np.array([len(w[3]) for w in want], np.int64)
    assert np.array_equal(np.diff(r.resp_off.astype(np.int64)), wl[pick])
    assert r.n_truncated == int(np.array([w[1] for w in want])[pick].sum())
    for i in np.random.default_rng(2).integers(0, len(pick), 50_000).tolist():
        w = want[pick[i]]
        assert (r.status[i], r.tc[i], r.node[i], r.response(i)) == (w[0], w[1], w[2], w[3])
