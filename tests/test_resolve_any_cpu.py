"""REGK_RESOLVE_ANY_FORM on the CPU: the restatement in resolve_any_util on hand-built cases (every TTL-precedence row of
the reference README's "About TTLs", duplicates, member order, the ignored top-level address, depth, number forms,
escaped names, bytes the grammar refuses), the README's own records (tests/golden/readme_records.json), the general
reader of regk_resolve_any.cuh compiled with g++ under AddressSanitizer against the restatement on every truncation and
single-byte mutation of a corpus of payloads placed flush against the end of their buffers, and the flag's value."""
import json
import os
import random
import re
import shutil
import subprocess
import tempfile

import pytest

import resolve_any_util as ra
import resolve_util as rv
from oracle import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = b"/us/joyent/example/b44c74d6"


def readme_records():
    with open(os.path.join(ROOT, "tests", "golden", "readme_records.json")) as f:
        return [(r["path"].encode(), r["data"].encode()) for r in json.load(f)["records"]]


def gen(data):
    return ra.general(data)


def host(typ=b"load_balancer", addr=b"10.0.0.1", inner_ttl=None, top_ttl=None, ports=None):
    inner = b'"address": "%s"' % addr + (b', "ttl": %s' % inner_ttl if inner_ttl is not None else b"") + (
        b', "ports": [%s]' % b", ".join(ports) if ports is not None else b"")
    return b'{\n "type": "%s",%s\n "%s": { %s }\n}' % (typ, b' "ttl": %s,' % top_ttl if top_ttl is not None else b"", typ, inner)


def service(sin_ttl=None, mid_ttl=None, top_ttl=None, port=b"80"):
    sin = b'"srvce": "_http", "proto": "_tcp", "port": %s' % port + (b', "ttl": %s' % sin_ttl if sin_ttl is not None else b"")
    mid = b'"type": "service", "service": { %s }' % sin + (b', "ttl": %s' % mid_ttl if mid_ttl is not None else b"")
    return b'{ "type": "service", "service": { %s }%s }' % (mid, b', "ttl": %s' % top_ttl if top_ttl is not None else b"")


def test_ttl_precedence_rows():
    # README.md "About TTLs": a host's A TTL is the inner ttl, else the top-level one
    assert gen(host(inner_ttl=b"10", top_ttl=b"20"))[3] == 10
    assert gen(host(top_ttl=b"20"))[3] == 20
    assert gen(host(inner_ttl=b"10"))[3] == 10
    assert gen(host())[3] is None
    # a service's SRV TTL: service.service.ttl, else service.ttl, else ttl
    assert gen(service(sin_ttl=b"1", mid_ttl=b"2", top_ttl=b"3"))[4] == 1
    assert gen(service(mid_ttl=b"2", top_ttl=b"3"))[4] == 2
    assert gen(service(sin_ttl=b"1", top_ttl=b"3"))[4] == 1
    assert gen(service(top_ttl=b"3"))[4] == 3
    assert gen(service())[4] is None
    # the A answer of a service name takes min(srv_ttl, a_ttl): README.md:752-755
    nodes = [(b"/s", service(mid_ttl=b"60")), (b"/s/h", host(typ=b"redis_host", top_ttl=b"30", ports=[b"1"]))]
    res = ra.resolve(nodes, 5, 7, True)
    assert res["sections"][0][0] == b"s.\t30\tIN\tA\t10.0.0.1\n"
    assert res["sections"][1] == (b"_http._tcp.s.\t60\tIN\tSRV\t0 10 1 h.s.\n", b"h.s.\t30\tIN\tA\t10.0.0.1\n")


def test_members_order_duplicates_address():
    assert gen(b'{"redis_host":{"ports":[1],"address":"1.2.3.4"},"ttl":5,"type":"redis_host"}') == (
        "host", b"redis_host", b"1.2.3.4", 5, [1])
    assert gen(b'{"type":"host","type":"db_host","db_host":{"address":"1.1.1.1"}}')[1] == b"db_host"
    assert gen(b'{"type":"host","host":{"address":"1.1.1.1"},"host":{"address":"2.2.2.2","address":"3.3.3.3"}}')[2] == b"3.3.3.3"
    assert gen(b'{"type":"host","host":{"address":"1.1.1.1","ports":[1]},"host":{"address":"2.2.2.2"}}')[4] is None
    assert gen(b'{"type":"host","host":{"address":"1.1.1.1"},"host":5}') is None
    # the top-level address is ignored: absent, different, of any type
    for top in (b"", b'"address":"9.9.9.9",', b'"address":null,', b'"address":{"x":[1]},'):
        assert gen(b'{"type":"host",%s"host":{"address":"1.1.1.1"}}' % top) == ("host", b"host", b"1.1.1.1", None, None)
    assert gen(b'{"type":"host","address":"1.1.1.1","host":{}}') is None
    assert gen(b'{"type":"host","host":{"address":"1.1.1.1","ports":[]}}')[4] == []
    for ports in (b"[1.0]", b"[-1]", b"[4294967296]", b'["1"]', b"[[1]]", b"1", b"null"):
        assert gen(b'{"type":"host","host":{"address":"1.1.1.1","ports":%s}}' % ports) is None
    assert gen(b'{"type":"host","host":{"address":"1.1.1.1","ports":[4294967295]}}')[4] == [2 ** 32 - 1]
    # a service's middle type is not required; srvce, proto, port are
    assert gen(b'{"type":"service","service":{"service":{"srvce":"_a","proto":"_b","port":1}}}') == ("service", b"_a", b"_b", 1, None)
    for drop in (b'"srvce":"_a",', b'"proto":"_b",'):
        assert gen(b'{"type":"service","service":{"service":{%s"port":1}}}' % b'"srvce":"_a","proto":"_b",'.replace(drop, b"")) is None
    # unknown members at any depth are skipped, but grammar-checked
    assert gen(b'{"x":[{"y":[1e5,-0.5,true,false,null,"\\u00e9"]}],"type":"host","host":{"address":"1.1.1.1","z":{}}}')
    assert gen(b'{"x":[1,],"type":"host","host":{"address":"1.1.1.1"}}') is None


def test_numbers():
    for bad in (b"-0", b"1e1", b"1.0", b"null", b'"30"', b"true", b"2147483648", b"-2147483649", b"[30]", b"{}"):
        assert gen(host(inner_ttl=bad)) is None, bad
        assert gen(host(top_ttl=bad, inner_ttl=b"5")) is None, bad      # every inspected ttl must be an integer
        assert gen(service(mid_ttl=bad, sin_ttl=b"5")) is None, bad
    assert gen(host(inner_ttl=b"-2147483648"))[3] == -2 ** 31
    assert gen(host(inner_ttl=b"2147483647"))[3] == 2 ** 31 - 1
    assert gen(service(port=b"4294967295"))[3] == 2 ** 32 - 1
    for bad in (b"4294967296", b"-1", b"80.0", b"8e1", b"-0", b"null"):
        assert gen(service(port=bad)) is None, bad
    # a ttl nested deeper than the inspected objects is skipped
    assert gen(b'{"type":"host","x":{"ttl":"no"},"host":{"address":"1.1.1.1","y":{"ttl":null}}}')[3] is None


def test_grammar_edges():
    ok = b'{"type":"host","host":{"address":"1.1.1.1"}}'
    assert gen(ok) and gen(b" \t\r\n" + ok + b"\n\n ")
    for bad in (b"\xef\xbb\xbf" + ok, ok + b"x", ok + b"{}", b"[" + ok + b"]", ok[:-1], b"", b" ", ok.replace(b":", b": :", 1),
                ok.replace(b'"1.1.1.1"', b'"1.1\x01.1"'), ok.replace(b'"1.1.1.1"', b'"1.1\n.1"'), ok + b"\x00",
                ok.replace(b'"type"', b'"ty\\u0070e"'), ok.replace(b'"host":{', b'"ho\\"st":{'), b"\xa0" + ok,
                ok.replace(b"1.1.1.1", b"1\\x")):
        assert gen(bad) is None, bad
    # bytes >= 0x80 inside strings are taken raw
    assert gen(ok.replace(b"1.1.1.1", b"1.1.1.\xff"))[2] == b"1.1.1.\xff"
    # escapes in values are kept as they are
    assert gen(ok.replace(b"1.1.1.1", b"1.1.1.\\u0031"))[2] == b"1.1.1.\\u0031"
    # an escaped member name anywhere refuses the payload
    assert gen(b'{"a":{"b\\n":1},"type":"host","host":{"address":"1.1.1.1"}}') is None


def nest(depth):
    """a host record with an unknown member whose value nests to `depth` containers in all (the top object counts)"""
    inner = b"[" * (depth - 1) + b"]" * (depth - 1)
    return b'{"type":"host","host":{"address":"1.1.1.1"},"x":%s}' % inner


def test_depth():
    assert gen(nest(64)) and gen(nest(65)) is None
    assert gen(nest(2))


def test_readme_records_verbatim():
    recs = readme_records()
    got = [ra.classify(p, d, True) for p, d in recs]
    assert got == [(rv.OK, ("service", b"_redis", b"_tcp", 6379, 60)),
                   (rv.OK, ("host", b"redis_host", b"172.27.10.62", 30, [6379])),
                   (rv.OK, ("host", b"redis_host", b"172.27.10.67", 30, [6379])),
                   (rv.OK, ("host", b"load_balancer", b"172.27.10.72", None, [80])),
                   (rv.OK, ("service", b"_http", b"_tcp", 80, 60))]
    assert all(ra.classify(p, d, False)[0] == rv.NOT_RECORD for p, d in recs)


def test_agreement_with_canonical(built):
    """for payloads the oracle composes, the general reader yields the canonical reader's record"""
    rng = random.Random(7)
    n = 0
    for _ in range(300):
        typ = rng.choice([b"load_balancer", b"redis_host", b"db_host", b"x_y"])
        addr = b"10.%d.%d.%d" % (rng.randrange(256), rng.randrange(256), rng.randrange(256))
        ttl = rng.choice([None, 0, 30, -5, 2 ** 31 - 1, -2 ** 31])
        ports = rng.choice([None, [], [rng.randrange(65536)], [1, 2, 3]])
        for data in (oracle.host_record_json(typ, addr, ttl, ports),
                     oracle.service_json(b"_s%d" % rng.randrange(9), b"_tcp", rng.randrange(65536), rng.choice([0, 60, -1]),
                                         tuple(rng.sample(range(4), 4)))):
            canon = rv.record(data)
            assert canon is not None and gen(data) == canon, data
            n += 1
    assert n == 600


def test_flag_values(built):
    from registrar_b200 import _native
    with open(os.path.join(ROOT, "include", "regk.h")) as f:
        h = f.read()
    m = re.search(r"#define REGK_RESOLVE_ANY_FORM \(1u << (\d+)\)", h)
    assert m and int(m.group(1)) == 12
    assert _native.FLAG_RESOLVE_ANY_FORM == 1 << 12
    taken = {int(x) for x in re.findall(r"#define REGK_\w+ +\(1u << (\d+)\)", h)}
    assert sorted(taken).count(12) == 1


# ------------------------------------------------------------------------------------------ the reader under ASan --

@pytest.fixture(scope="module")
def any_emul(built):
    if not shutil.which("g++"):
        pytest.skip("g++ not available")
    d = tempfile.mkdtemp(prefix="regk_any_emul_")
    exe = os.path.join(d, "resolve_any_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=undefined", "-o", exe, os.path.join(ROOT, "tests", "emul", "resolve_any_emul.cpp")])
    yield exe
    shutil.rmtree(d, ignore_errors=True)


def expected(path, data, dh, ds):
    """the emul's line for one node, from the restatement"""
    c, rec = ra.classify(path, data, True)
    _, g = ra.record(path, data, True)
    read = 1 if g is not None else 0
    if c in (rv.EMPTY, rv.NOT_RECORD):
        return "%d 0 0 %d - - - 0 -" % (c, read)
    svc = rec[0] == "service"
    ttl = rec[4] if svc else rec[3]
    ttl = (ds if svc else dh) if ttl is None else ttl
    roles = 0
    if c == rv.OK:
        roles = 2 if svc else (1 if rec[1] in rv.QUERYABLE else 0) | (4 if rec[1] in rv.USABLE else 0)
    ports = [rec[3]] if svc else rec[4]
    return "%d %d %d %d %s %s %s %d %s" % (c, roles, ttl, read, "s" if svc else "h", rec[1].hex() or "-", rec[2].hex() or "-",
                                           -1 if ports is None else len(ports),
                                           ",".join(str(p) for p in ports) if ports else "-")


def run_emul(exe, cases):
    inp = "".join("%s %s %d %d\n" % (p.hex() or "-", d.hex() or "-", dh, ds) for p, d, dh, ds in cases)
    out = subprocess.run([exe], input=inp.encode(), capture_output=True)
    assert out.returncode == 0, out.stderr.decode()[-3000:]
    got = out.stdout.decode().splitlines()
    assert len(got) == len(cases)
    for (p, d, dh, ds), line in zip(cases, got):
        assert line == expected(p, d, dh, ds), (p, d, line)


def corpus():
    c = [d for _, d in readme_records()]
    c += [host(inner_ttl=b"10", top_ttl=b"-20", ports=[b"1", b"65536"]), service(sin_ttl=b"1", mid_ttl=b"2", top_ttl=b"3"),
          b'{"redis_host":{"ports":[1,2],"address":"1.2.3.4","ttl":7},"ttl":5,"type":"redis_host","z":[{"a":1e-3}]}',
          b'{"type":"host","host":{"address":"1.1.1.\\u0031"},"x":"\\"\\\\\\/\\b\\f\\n\\r\\t"}',
          nest(64), b'{"type":"se\\u0072vice","service":{}}', b'{"type":"service","service":{"service":{"srvce":"_a b",'
          b'"proto":"_tcp","port":4294967295,"ttl":-2147483648}},"ttl":true}',
          oracle.host_record_json(b"redis_host", b"10.1.2.3", 30, [6379]), oracle.service_json(b"_redis", b"_tcp", 6379, 60),
          oracle.host_record_json(b"load_balancer", b"10.1.2.3", None, None)]
    return c


def test_reader_asan_corpus(any_emul):
    cases = [(P, d, 30, 60) for d in corpus()]
    cases += [(b"/s", d, 1, 2) for d in corpus()] + [(b"", b"{}", 0, 0), (b"/x", b"", 0, 0), (b"x", corpus()[0], 0, 0)]
    run_emul(any_emul, cases)


def canonical_outside_model(d):
    """a canonical-form payload with control bytes, bytes >= 0x80 or a bad escape in its strings: the canonical reader
    accepts it (it skips escapes unread), resolve_util's restatement of that reader (json.loads on UTF-8) does not
    model it"""
    def plain(b):
        return 0x20 <= b < 0x80 and b != 0x5C
    if rv.record(d) is not None or all(plain(b) for b in d):
        return False
    return rv.record(bytes(b if plain(b) else 0x61 for b in d)) is not None


def test_reader_asan_truncations_and_mutations(any_emul):
    subst = b'{}[]",:\\ 0-1e.tnx\x00\x1f\x80\xff'
    cases = []
    for d in corpus():
        cases += [(P, d[:k], 30, 60) for k in range(len(d))]
        for k in range(len(d)):
            for b in subst:
                m = d[:k] + bytes([b]) + d[k + 1:]
                if d[k] != b and not canonical_outside_model(m):
                    cases.append((P, m, 30, 60))
    run_emul(any_emul, cases)
