"""regk_resolve on the CPU: the restatement in resolve_util against the reference README's worked dig outputs (nodes
composed by the composer oracle), the C-ABI struct layouts, and the per-node rules of regk_resolve.cuh compiled with g++
under AddressSanitizer against the restatement at every boundary of the name, address, ttl and port checks."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import pytest

import resolve_util as rv
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def host_node(domain, host, type_, addr, ttl=None, ports=None):
    return (oracle.host_node_path(domain, host), oracle.host_record_json(type_, addr, ttl, ports))


def alias_node(alias, type_, addr, ttl=None, ports=None):
    return (oracle.domain_to_path(alias), oracle.host_record_json(type_, addr, ttl, ports))


def service_node(domain, srvce, proto, port, ttl=60):
    return (oracle.domain_to_path(domain), oracle.service_json(srvce, proto, port, ttl))


AUTHCACHE = b"authcache.emy-10.joyent.us"
AC1, AC2 = b"a2674d3b-a9c4-46bc-a835-b6ce21d522c2", b"a4ae094d-da07-4911-94f9-c982dc88f3cc"


def readme_scenarios():
    """name -> snapshot nodes of the README's scenarios"""
    ex = b"example.joyent.us"
    plain = [host_node(ex, b"b44c74d6", b"load_balancer", b"172.27.10.72"),
             alias_node(b"host-1a." + ex, b"load_balancer", b"172.27.10.72"),
             alias_node(b"host-1b." + ex, b"load_balancer", b"172.27.10.72")]
    svc = [service_node(ex, b"_http", b"_tcp", 80), host_node(ex, b"b44c74d6", b"load_balancer", b"172.27.10.72")]
    svc2 = svc + [host_node(ex, b"c5e0d7a1", b"load_balancer", b"172.27.10.73", ports=[80])]
    auth = [service_node(AUTHCACHE, b"_redis", b"_tcp", 6379),
            host_node(AUTHCACHE, AC1, b"redis_host", b"172.27.10.62", 30, [6379]),
            host_node(AUTHCACHE, AC2, b"redis_host", b"172.27.10.67", 30, [6379])]
    return {"plain": plain, "service": svc, "service2": svc2, "authcache": auth}


def lines(b):
    return sorted(tuple(x.split()) for x in b.decode().splitlines())


def by_query(res, nodes):
    """(kind, name) -> (answer, additional)"""
    out = {}
    for q, (kind, j) in enumerate(zip(res["q_kind"], res["q_node"])):
        out[(kind, rv.name_of(nodes[j][0]))] = res["sections"][q]
    return out


def check_readme(get):
    """get(nodes) -> {(kind, name): (answer, additional)}; the README's dig lines, as sets where the order is Binder's"""
    sc = readme_scenarios()
    ex = b"example.joyent.us"
    got = get(sc["plain"])
    for host in (b"host-1a", b"host-1b", b"b44c74d6"):              # README.md:342-347 (+short: the address)
        ans = got[(rv.HOST_A, host + b"." + ex)][0]
        assert [x.split()[-1] for x in ans.decode().splitlines()] == ["172.27.10.72"]
    assert (rv.SERVICE_A, ex) not in got                            # no service record: nothing lists the hosts
    got = get(sc["service"])
    assert got[(rv.HOST_A, b"b44c74d6." + ex)][0].split()[-1] == b"172.27.10.72"    # README.md:409-410
    assert [x.split()[-1] for x in got[(rv.SERVICE_A, ex)][0].splitlines()] == [b"172.27.10.72"]    # :415-416
    srv, add = got[(rv.SERVICE_SRV, ex)]                            # README.md:432-433 and :705-708
    assert lines(srv) == lines(b"_http._tcp.example.joyent.us. 60 IN     SRV     0 10 80 b44c74d6.example.joyent.us.\n")
    assert lines(add) == lines(b"b44c74d6.example.joyent.us. 30  IN      A       172.27.10.72\n")
    got = get(sc["service2"])                                       # README.md:420-422
    assert sorted(x.split()[-1] for x in got[(rv.SERVICE_A, ex)][0].splitlines()) == [b"172.27.10.72", b"172.27.10.73"]
    got = get(sc["authcache"])
    # README.md:223 and :573
    assert lines(got[(rv.HOST_A, AC1 + b"." + AUTHCACHE)][0]) == lines(
        b"a2674d3b-a9c4-46bc-a835-b6ce21d522c2.authcache.emy-10.joyent.us. 30 IN A 172.27.10.62\n")
    # README.md:232-233 and :564-565
    assert lines(got[(rv.SERVICE_A, AUTHCACHE)][0]) == lines(
        b"authcache.emy-10.joyent.us. 30  IN      A       172.27.10.67\n"
        b"authcache.emy-10.joyent.us. 30  IN      A       172.27.10.62\n")
    assert got[(rv.SERVICE_A, AUTHCACHE)][1] == b""


def test_readme_vectors_restated(built):
    check_readme(lambda nodes: by_query(rv.resolve(nodes, 30, 60), nodes))


def test_restatement_worked_by_hand():
    nodes = [(b"/us/x", b'{"type":"service","service":{"type":"service","service":{"srvce":"_a","proto":"_udp","port":53}}}'),
             (b"/us/x/h1", b'{"type":"rr_host","address":"10.0.0.1","ttl":5,"rr_host":{"address":"10.0.0.1","ports":[1,2]}}'),
             (b"/us/x/h2", b'{"type":"rr_host","address":"10.0.0.2","rr_host":{"address":"10.0.0.2","ports":[]}}'),
             (b"/us/x/h3", b'{"type":"host","address":"10.0.0.3","host":{"address":"10.0.0.3"}}'),
             (b"/us", b"")]
    r = rv.resolve(nodes, 30, 60)
    assert r["q_kind"] == [rv.SERVICE_A, rv.SERVICE_SRV, rv.HOST_A] and r["q_node"] == [0, 0, 3]
    assert r["sections"][0] == (b"x.us.\t5\tIN\tA\t10.0.0.1\nx.us.\t30\tIN\tA\t10.0.0.2\n", b"")
    assert r["sections"][1] == (b"_a._udp.x.us.\t60\tIN\tSRV\t0 10 1 h1.x.us.\n_a._udp.x.us.\t60\tIN\tSRV\t0 10 2 h1.x.us.\n",
                                b"h1.x.us.\t5\tIN\tA\t10.0.0.1\n")
    assert r["node_cls"] == [rv.OK] * 4 + [rv.EMPTY] and r["unresolved"] == []
    assert (r["n_answers"], r["n_additional"]) == (5, 1)
    with pytest.raises(rv.DuplicateNode) as e:
        rv.resolve(nodes + [(b"/us/x/h2", b"")], 30, 60)
    assert e.value.node == 5


def test_struct_layouts_match_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu ", sizeof(regk_resolve_opts), offsetof(regk_resolve_opts, default_host_ttl),
               offsetof(regk_resolve_opts, default_srv_ttl), offsetof(regk_resolve_opts, reserved), sizeof(regk_answers));
        printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu ", offsetof(regk_answers, n_queries),
               offsetof(regk_answers, n_unresolved), offsetof(regk_answers, text_total), offsetof(regk_answers, flags),
               offsetof(regk_answers, launches), offsetof(regk_answers, q_kind), offsetof(regk_answers, q_node),
               offsetof(regk_answers, sec_off), offsetof(regk_answers, text), offsetof(regk_answers, node_cls),
               offsetof(regk_answers, unresolved), offsetof(regk_answers, kernel_ms));
        printf("%u %u %u %u %u\n", REGK_Q_HOST_A, REGK_Q_SERVICE_SRV, REGK_RSV_EMPTY, REGK_RSV_BAD_ADDRESS, REGK_RSV_BAD_PORT);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    O, A = _native.CResolveOpts, _native.CAnswers
    assert got == [C.sizeof(O), O.default_host_ttl.offset, O.default_srv_ttl.offset, O.reserved.offset, C.sizeof(A),
                   A.n_queries.offset, A.n_unresolved.offset, A.text_total.offset, A.flags.offset, A.launches.offset,
                   A.q_kind.offset, A.q_node.offset, A.sec_off.offset, A.text.offset, A.node_cls.offset,
                   A.unresolved.offset, A.kernel_ms.offset, _native.Q_HOST_A, _native.Q_SERVICE_SRV, _native.RSV_EMPTY,
                   _native.RSV_BAD_ADDRESS, _native.RSV_BAD_PORT]
    assert "regk_resolve" in _native.EXPORTS


@pytest.fixture(scope="module")
def emul(built):
    d = tempfile.mkdtemp(prefix="regk_resolve_emul")
    exe = os.path.join(d, "resolve_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "resolve_emul.cpp")])

    def run(cases, dh=30, ds=60):
        """cases = [(path, data)] -> [(class, roles, ttl, line)]"""
        inp = "".join("%s %s %d %d\n" % (p.hex() or "-", j.hex() or "-", dh, ds) for p, j in cases)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input=inp, capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        out = []
        for ln in p.stdout.splitlines():
            c, r, t, h = ln.split()
            out.append((int(c), int(r), int(t), b"" if h == "-" else bytes.fromhex(h)))
        return out
    yield run
    shutil.rmtree(d, ignore_errors=True)


def want(path, data, dh=30, ds=60):
    """the restatement's (class, roles, ttl, line) for one node, as the emulator reports it"""
    c, rec = rv.classify(path, data)
    if c != rv.OK:
        return c, 0, None, b""
    name = rv.name_of(path)
    if rec[0] == "service":
        ttl = ds if rec[4] is None else rec[4]
        return c, 2, ttl, rv.srv_line(rec[1], rec[2], name, ttl, rec[3], b"c.x")
    ttl = dh if rec[3] is None else rec[3]
    roles = (1 if rec[1] in rv.QUERYABLE else 0) | (4 if rec[1] in rv.USABLE else 0)
    return c, roles, ttl, rv.a_line(name, ttl, rec[2]) if roles & 1 else b""


def host(typ=b"host", addr=b"10.1.2.3", ttl=None, ports=None, key=None, addr2=None):
    out = b'{"type":"%s","address":"%s"' % (typ, addr)
    if ttl is not None:
        out += b',"ttl":%s' % (ttl if isinstance(ttl, bytes) else str(ttl).encode())
    out += b',"%s":{"address":"%s"' % (key or typ, addr2 or addr)
    if ports is not None:
        out += b',"ports":[' + b",".join(str(p).encode() for p in ports) + b"]"
    return out + b"}}"


def service(srvce=b"_http", proto=b"_tcp", port=80, ttl=60):
    inner = b'"srvce":"%s","proto":"%s","port":%d' % (srvce, proto, port)
    if ttl is not None:
        inner += b',"ttl":%d' % ttl
    return b'{"type":"service","service":{"type":"service","service":{' + inner + b"}}}"


def boundary_cases():
    l63, l64 = b"a" * 63, b"b" * 64
    cases = []
    for lab in (l63, l64, b"x_y-Z9", b"x.y", b"x*y", b"\xc3\xa9"):
        cases.append((b"/com/" + lab, host()))
    for n in (253, 254):                                            # whole names of 253 and 254 bytes
        labels, rest = [], n
        while rest > 0:
            k = min(63, rest)
            labels.append(b"c" * k)
            rest -= k + 1
        name = b".".join(labels)[:n]
        if name.endswith(b"."):
            name = name[:-1] + b"d"
        assert len(name) == n
        cases.append((b"/" + b"/".join(reversed(name.split(b"."))), host()))
        cases.append((b"/" + b"/".join(reversed(name.split(b".")[1:])), service(srvce=b"_" + b"s" * 10)))
    for addr in (b"255.255.255.255", b"256.1.1.1", b"010.1.1.1", b"0.0.0.0", b"1.2.3", b"1.2.3.4.5", b"1..3.4", b"1.2.3.4 ",
                 b"", b"1234.1.1.1", b"a.b.c.d"):
        cases.append((b"/com/h", host(addr=addr)))
    for ttl in (0, -1, 2 ** 31 - 1, -2 ** 31, 2 ** 31, b"-0", b"01", b"1.5"):
        cases.append((b"/com/h", host(ttl=ttl)))
    for ttl in (0, -1, 2 ** 31 - 1, -2 ** 31, None):
        cases.append((b"/com/s", service(ttl=ttl)))
    for ports in ([65535], [65536], [], [1, 65536, 2], [2 ** 32 - 1], [2 ** 32]):
        cases.append((b"/com/h", host(typ=b"rr_host", ports=ports)))
    for port in (0, 65535, 65536):
        cases.append((b"/com/s", service(port=port)))
    for typ in (b"db_host", b"host", b"load_balancer", b"moray_host", b"ops_host", b"redis_host", b"rr_host", b"service",
                b"database", b"hos\\u0074", b"", b"ttl", b"address"):
        cases.append((b"/com/h", host(typ=typ)))
    cases += [(b"/com/h", host(key=b"host2")), (b"/com/h", host(addr2=b"10.1.2.4")), (b"/com/h", b""), (b"", host()),
              (b"com/h", host()), (b"/", host()), (b"/com//h", host()), (b"/com/h/", host()),
              (b"/com/s", service(srvce=b"_ht\\\"tp")), (b"/com/s", service(srvce=b"")), (b"/com/s", service(srvce=b"a.b")),
              (b"/com/s", service(proto=b"_" + b"p" * 63)), (b"/com/h", b'{"type": "host"}'), (b"/com/h", b"null"),
              (b"/com/h", b'{"type":"host","address":"1.2.3.4","host":{"address":"1.2.3.4"}} ')]
    return cases


def test_rules_at_every_boundary(emul):
    cases = boundary_cases()
    got = emul(cases)
    for (path, data), g in zip(cases, got):
        w = want(path, data)
        assert g[:2] == w[:2] and (w[2] is None or g[2] == w[2]) and g[3] == w[3], (path, data, g, w)
    classes = {want(p, d)[0] for p, d in cases}
    assert classes == set(range(8))


def test_default_ttls_reach_the_lines(emul):
    cases = [(b"/com/h", host()), (b"/com/s", service(ttl=None))]
    got = emul(cases, dh=0, ds=2 ** 31 - 1)
    assert [g[2] for g in got] == [0, 2 ** 31 - 1]
    assert got[1][3] == rv.srv_line(b"_http", b"_tcp", b"s.com", 2 ** 31 - 1, 80, b"c.x")
