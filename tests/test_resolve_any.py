"""REGK_RESOLVE_ANY_FORM on the GPU, bit for bit against the restatement in resolve_any_util: the reference README's
records pasted verbatim (tests/golden/readme_records.json), random mixed snapshots of canonical, general and broken
payloads from host and device snapshots with host and device outputs, flag-off parity on canonical snapshots, DNS
answers (with and without PTR) after a flagged resolve, a watched walk of the README tree with verbatim payloads, a
device snapshot whose last payload ends at the tensor's end, and a fleet of 4 M pretty-printed, reordered host records
under 1 000 services against the same records composed canonically."""
import json
import random

import numpy as np
import pytest

import dns_ptr_util as pu
import dns_util as du
import resolve_any_util as ra
import resolve_util as rv
from test_dns import compare as dns_compare, host_dict
from test_reconcile import device_snapshot
from test_resolve import compare, host_snapshot, raw_to_dict, random_snapshot
from test_resolve_any_cpu import readme_records
from test_resolve_cpu import AC1, AC2, AUTHCACHE, check_readme, lines

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def every_way(ctx, nodes, dh=30, ds=60, any_form=True):
    """host and device snapshots, host and device outputs, all against the restatement; returns the host Answers"""
    want = ra.resolve(nodes, dh, ds, any_form)
    got = ctx.resolve(host_snapshot(nodes), dh, ds, any_form=any_form)
    compare(got, want)
    dsnap = device_snapshot(nodes)
    compare(ctx.resolve(dsnap, dh, ds, any_form=any_form), want)
    compare(raw_to_dict(ctx, ctx.resolve(dsnap, dh, ds, device=True, any_form=any_form)), want)
    compare(raw_to_dict(ctx, ctx.resolve(host_snapshot(nodes), dh, ds, device=True, any_form=any_form)), want)
    return got


def readme_nodes():
    """the README's records verbatim at the README's paths, with their directories"""
    recs = readme_records()
    dirs = [(b"/us", b""), (b"/us/joyent", b""), (b"/us/joyent/emy-10", b"")]
    return dirs + recs


def test_readme_records_answer_as_the_readme_shows(ctx):
    nodes = readme_nodes()
    a = every_way(ctx, nodes)
    assert a.node_cls.tolist() == [rv.EMPTY] * 3 + [rv.OK] * 5
    got = {(int(k), rv.name_of(nodes[int(j)][0])): (a.answer(q), a.additional(q)) for q, (k, j) in enumerate(zip(a.q_kind, a.q_node))}
    # README.md:223 and :573: the instances' A answers, TTL 30
    assert lines(got[(rv.HOST_A, AC1 + b"." + AUTHCACHE)][0]) == lines(
        b"a2674d3b-a9c4-46bc-a835-b6ce21d522c2.authcache.emy-10.joyent.us. 30 IN A 172.27.10.62\n")
    # the service's A answers take min(srv_ttl 60, a_ttl 30); its SRV answers TTL 60 (the middle-level ttl of the
    # README's record and the inner one agree), additionals 30
    assert lines(got[(rv.SERVICE_A, AUTHCACHE)][0]) == lines(
        b"authcache.emy-10.joyent.us. 30 IN A 172.27.10.62\nauthcache.emy-10.joyent.us. 30 IN A 172.27.10.67\n")
    srv, add = got[(rv.SERVICE_SRV, AUTHCACHE)]
    assert lines(srv) == lines(b"_redis._tcp.authcache.emy-10.joyent.us. 60 IN SRV 0 10 6379 %s.authcache.emy-10.joyent.us.\n"
                               b"_redis._tcp.authcache.emy-10.joyent.us. 60 IN SRV 0 10 6379 %s.authcache.emy-10.joyent.us.\n"
                               % (AC1, AC2))
    assert lines(add) == lines(b"%s.authcache.emy-10.joyent.us. 30 IN A 172.27.10.62\n"
                               b"%s.authcache.emy-10.joyent.us. 30 IN A 172.27.10.67\n" % (AC1, AC2))
    # README.md:409-433 and :705-708 with the README's _http service and load_balancer host as written
    ex = b"example.joyent.us"
    assert lines(got[(rv.SERVICE_SRV, ex)][0]) == lines(b"_http._tcp.example.joyent.us. 60 IN SRV 0 10 80 b44c74d6.example.joyent.us.\n")
    assert lines(got[(rv.SERVICE_SRV, ex)][1]) == lines(b"b44c74d6.example.joyent.us. 30 IN A 172.27.10.72\n")
    assert got[(rv.HOST_A, b"b44c74d6." + ex)][0].split()[-1] == b"172.27.10.72"
    # without the flag: today's NOT_RECORD for every one of them
    off = every_way(ctx, nodes, any_form=False)
    assert off.node_cls.tolist() == [rv.EMPTY] * 3 + [rv.NOT_RECORD] * 5 and off.n_queries == 0


def pretty(data: bytes, rng) -> bytes:
    """a canonical payload in another layout: members reordered at every level, indented (json.dumps keeps ASCII
    strings as they are)"""
    def shuffle(v):
        if isinstance(v, dict):
            items = list(v.items())
            rng.shuffle(items)
            return {k: shuffle(x) for k, x in items}
        return v
    return json.dumps(shuffle(json.loads(data)), indent=rng.choice([None, 1, 2, 4]),
                      separators=rng.choice([None, (",", ":"), (", ", ": ")])).encode()


def test_readme_scenarios_in_any_layout(ctx):
    rng = random.Random(2)

    def get(nodes):
        nodes = [(p, pretty(d, rng) if d else d) for p, d in nodes]
        a = every_way(ctx, nodes)
        return {(int(k), rv.name_of(nodes[int(j)][0])): (a.answer(q), a.additional(q)) for q, (k, j) in enumerate(zip(a.q_kind, a.q_node))}
    check_readme(get)


def general_payload(rng):
    """a general-form payload of every kind the rules name, ASCII strings only"""
    typ = rng.choice([b"db_host", b"host", b"load_balancer", b"moray_host", b"ops_host", b"redis_host", b"rr_host", b"nope"])
    addr = rng.choice([b"10.%d.%d.%d" % (rng.randrange(256), rng.randrange(256), rng.randrange(256))] * 6 + [b"1.2.3", b"01.1.1.1"])
    ttl = lambda: rng.choice([b"30", b"0", b"-5", b"3600", b"1.0", b"null", b"-0", b"2147483647"] + [None] * 6)
    r = rng.random()
    if r < 0.45:
        inner = [b'"address": "%s"' % addr]
        t = ttl()
        if t is not None:
            inner.append(b'"ttl": %s' % t)
        if rng.random() < 0.6:
            inner.append(b'"ports": [%s]' % b", ".join(b"%d" % rng.choice([80, 6379, 65535, 65536]) for _ in range(rng.randrange(4))))
        rng.shuffle(inner)
        top = [b'"type": "%s"' % typ, b'"%s": {%s}' % (typ, b", ".join(inner))]
        if rng.random() < 0.5:
            top.append(b'"address": "%s"' % rng.choice([addr, b"9.9.9.9"]))
        t = ttl()
        if t is not None:
            top.append(b'"ttl": %s' % t)
        if rng.random() < 0.2:
            top.append(b'"extra": {"ttl": "x", "a": [1e3, true, {"b": null}]}')
        rng.shuffle(top)
        return b"{\n  " + b",\n  ".join(top) + b"\n}\n"
    if r < 0.85:
        sin = [b'"srvce": "%s"' % rng.choice([b"_http", b"_redis", b"_a b"]), b'"proto": "_tcp"',
               b'"port": %s' % rng.choice([b"80", b"65535", b"65536", b"8.0"])]
        mid = [b'"service": {%s}' % b", ".join(sin)]
        top = [b'"type": "service"', b'"service": {%s}' % b", ".join(mid)]
        for lst in (sin, mid, top):
            t = ttl()
            if t is not None:
                lst.append(b'"ttl": %s' % t)
        mid.append(b'"type": "service"')
        mid[0] = b'"service": {%s}' % b", ".join(sin)
        top[1] = b'"service": {%s}' % b", ".join(mid)
        rng.shuffle(top)
        return b"{ " + b", ".join(top) + b" }"
    return rng.choice([b'{"type":"host"}', b"[1]", b'{"type":"host","host":{"address":"1.1.1.1"}} x', b"{", b"null",
                       b'{"type":"host","ho\\u0073t":{"address":"1.1.1.1"}}'])


def mixed_snapshot(rng):
    nodes = random_snapshot(rng)
    seen = {p for p, _ in nodes}
    out = []
    for p, d in nodes:
        if d and rng.random() < 0.4:
            d = general_payload(rng)
        elif d and rng.random() < 0.2:
            try:
                d = pretty(d, rng)
            except ValueError:
                pass
        out.append((p, d))
    for k in range(rng.randrange(3, 12)):                   # general records under the existing directories
        base = rng.choice([p for p, _ in nodes])
        p = base + b"/g%d" % k
        if p not in seen:
            seen.add(p)
            out.append((p, general_payload(rng)))
    return out


@pytest.mark.parametrize("seed", range(6))
def test_random_mixed_snapshots(ctx, seed):
    rng = random.Random(seed)
    nodes = mixed_snapshot(rng)
    a = every_way(ctx, nodes, rng.choice([0, 30]), rng.choice([0, 60]))
    every_way(ctx, nodes, 30, 60, any_form=False)
    assert a.m == len(nodes)


def test_canonical_snapshot_same_with_and_without_the_flag(ctx):
    rng = random.Random(11)
    nodes = [(p, d) for p, d in random_snapshot(rng) if not d or rv.record(d) is not None]
    on = ctx.resolve(host_snapshot(nodes), 30, 60, any_form=True)
    off = ctx.resolve(host_snapshot(nodes), 30, 60)
    for k in ("q_kind", "q_node", "sec_off", "text", "node_cls", "unresolved"):
        assert np.array_equal(getattr(on, k), getattr(off, k)), k
    assert on.launches == off.launches + 2                  # count and compaction; no candidate, no reader
    nodes.append((b"/zz", b'{ "type": "host", "host": { "address": "1.2.3.4" } }'))
    assert ctx.resolve(host_snapshot(nodes), 30, 60, any_form=True).launches == off.launches + 3


def test_dns_after_a_flagged_resolve(ctx):
    rng = random.Random(5)
    for _ in range(3):
        nodes = mixed_snapshot(rng)
        zone = du.Zone(ra.restated(nodes, True))
        ctx.resolve(host_snapshot(nodes), 30, 60, any_form=True)
        names = [rv.name_of(p) for p, _ in nodes]
        msgs = [du.query(n, rng.choice([du.T_A, du.T_SRV, du.T_ANY])) for n in names]
        for j in zone.srv:
            _, srvce, proto, _, _ = zone.rec[j]
            if rv.valid_name(srvce + b"." + proto):
                msgs.append(du.query(srvce + b"." + proto + b"." + rv.name_of(nodes[j][0]), du.T_SRV))
        addrs = sorted(pu.reverse_map(zone))
        msgs += [du.query(pu.reverse_name(x), pu.T_PTR) for x in addrs] + [du.query(pu.reverse_name(b"10.255.255.254"), pu.T_PTR)]
        mb, mo = du.pack(msgs)
        dns_compare(host_dict(ctx.answer_dns(mb, mo)), du.answer_all(zone, msgs), msgs)
        dns_compare(host_dict(ctx.answer_dns(mb, mo, ptr=True)), pu.answer_all(zone, msgs), msgs)


def test_device_snapshot_ending_at_the_tensor_end(ctx):
    """the last payload is the last byte of the data tensor: the reader's bounded path"""
    import torch
    from registrar_b200.batch import Snapshot
    for last in (b'{"type":"host","host":{"address":"10.0.0.1"}}', b'{ "host": { "address": "10.0.0.1" }, "type": "host" }',
                 b'{"type":"host","host":{"address":"10.0.0.1"}', b'{"type":"service","service":{"service":{"srvce":"_a",'
                 b'"proto":"_b","port":1,"ttl":7}}}'):
        nodes = [(b"/a", b""), (b"/a/b", b'{"type":"host","ttl":5,"host":{"address":"10.0.0.2"}}'), (b"/a/c", last)]
        h = Snapshot.from_nodes(nodes)
        jb = torch.from_numpy(h.json_bytes.copy()).cuda()
        assert jb.numel() == len(b"".join(d for _, d in nodes))
        t = lambda a, dt: torch.from_numpy(a.view(dt)).cuda()
        snap = Snapshot(t(h.path_bytes, np.uint8), t(h.path_off, np.int64), jb, t(h.json_off, np.int64))
        compare(ctx.resolve(snap, 30, 60, any_form=True), ra.resolve(nodes, 30, 60, True))


def test_watched_walk_of_the_readme_tree(built):
    import walk_watch_util as ww
    from registrar_b200 import _native
    c, c2 = _native.Context(0), _native.Context(0)
    session = 3
    try:
        zk = ww.WalkZooKeeper()
        for p, d in readme_nodes():
            for k in range(1, p.count(b"/")):
                q = b"/".join(p.split(b"/")[:k + 1])
                if q not in zk.nodes:
                    zk.create(q, b"", 0, False)
            if p in zk.nodes:
                zk.set_data(p, d)
            else:
                zk.create(p, d, 0, False)
        zk.take_events(session)
        c.walk([b"/us"], lambda fb: zk.serve(fb, session), watch=True)

        def check(any_form, full):
            w = c.walk_resolve(30, 60, any_form=any_form)
            assert w.full == full
            snap = c._walk.snapshot()
            pb, po, jb, jo = snap.path_bytes.tobytes(), snap.path_off, snap.json_bytes.tobytes(), snap.json_off
            nodes = [(pb[po[j]:po[j + 1]], jb[jo[j]:jo[j + 1]]) for j in range(len(po) - 1)]
            want = ra.resolve(nodes, 30, 60, any_form)
            compare(w, want)
            plain = c2.resolve(host_snapshot(nodes), 30, 60, any_form=any_form)
            assert plain.text.tobytes() == w.text.tobytes()
            return w

        w = check(True, 1)
        assert w.n_queries == 7                     # three HOST_A names, two services' A and SRV
        check(True, 0)
        check(False, 1)                                     # toggling the flag formats everything
        check(False, 0)
        check(True, 1)
        # a refresh: one instance readdressed (pretty-printed still), one created; reuse stays exact
        zk.set_data(b"/us/joyent/emy-10/authcache/" + AC1, readme_records()[1][1].replace(b"172.27.10.62", b"172.27.10.99"))
        zk.create(b"/us/joyent/emy-10/authcache/n1", b'{\n "redis_host": { "address": "10.0.0.7", "ports": [ 6380 ] },\n'
                                                    b' "type": "redis_host"\n}', 0, False)
        c.walk_events(np.frombuffer(zk.take_events(session), np.uint8))
        c.refresh_walk(lambda fb: zk.serve(fb, session))
        w = check(True, 0)
        assert 0 < w.copied_bytes < w.text_total and w.n_fresh >= 2
    finally:
        c.close()
        c2.close()


@pytest.mark.slow
def test_fleet_four_million_pretty_printed_hosts(ctx):
    """4 M config 2 host records under 1 000 services: every payload pretty-printed and reordered, resolved with the
    flag, against the same records as composed resolved without it; then A, SRV and PTR responses"""
    import torch
    from registrar_b200.batch import Snapshot
    from test_resolve import fleet_nodes, fleet_snapshot
    got, idx = fleet_nodes(4_000_000)
    pb, po, jb, jo = fleet_snapshot(got, idx, 1000)
    m = len(po) - 1
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a).view(dt)).cuda()
    canon = Snapshot(t(pb, np.uint8), t(po, np.int64), t(jb, np.uint8), t(jo, np.int64))
    rng = random.Random(9)
    jbs = jb.tobytes()
    pieces = []
    for j in range(m):
        d = jbs[jo[j]:jo[j + 1]]
        pieces.append(pretty(d, rng) if j % 50 == 0 else
                      b"{\n  " + d[1:-1].replace(b',"', b',\n  "').replace(b'":', b'": ') + b"\n}\n")
    jb2 = np.frombuffer(b"".join(pieces), np.uint8)
    jo2 = np.zeros(m + 1, np.uint64)
    np.cumsum([len(x) for x in pieces], out=jo2[1:])
    gen = Snapshot(t(pb, np.uint8), t(po, np.int64), t(jb2, np.uint8), t(jo2, np.int64))
    want = ctx.resolve(canon, 30, 60)
    assert want.n_unresolved == 0
    a = ctx.resolve(gen, 30, 60, any_form=True)
    for k in ("q_kind", "q_node", "sec_off", "text", "node_cls", "unresolved"):
        assert np.array_equal(getattr(a, k), getattr(want, k)), k
    assert ctx.resolve(gen, 30, 60).n_unresolved >= m - m // 50   # json.dumps may give back a compact record in order
    # the same DNS responses, with and without PTR
    pbs = pb.tobytes()
    sample = rng.sample(range(m), 3000)
    names = [rv.name_of(pbs[po[j]:po[j + 1]]) for j in sample]
    addrs = [b"10.%d.%d.%d" % (rng.randrange(256), rng.randrange(256), rng.randrange(256)) for _ in range(500)]
    msgs = [du.query(n, rng.choice([du.T_A, du.T_SRV])) for n in names] + [du.query(pu.reverse_name(x), pu.T_PTR) for x in addrs]
    mb, mo = du.pack(msgs)
    out = {}
    for flag, snap in ((False, canon), (True, gen)):
        ctx.resolve(snap, 30, 60, any_form=flag)
        out[flag] = (host_dict(ctx.answer_dns(mb, mo)), host_dict(ctx.answer_dns(mb, mo, ptr=True)))
    assert out[False] == out[True]
    assert sum(1 for s in out[True][1]["status"] if s == du.ANSWER) > 1000
