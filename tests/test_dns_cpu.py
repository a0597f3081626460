"""regk_dns_answer on the CPU: the message parser, the question's path and the truncation arithmetic of regk_dns.cuh
compiled with g++ under AddressSanitizer against the restatement in dns_util (every truncation point of valid
queries, every single-byte mutation of the header, counts and labels, label lengths 63 / 64, names of 255 / 256 wire
bytes, pointers and extended labels, OPT variants); the restatement's responses decoded by dnspython; the C-ABI
struct layouts."""
import ctypes as C
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import dns_util as du
import resolve_util as rv
from test_resolve_cpu import host, readme_scenarios, service

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_struct_layouts_match_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu ", sizeof(regk_dns_in), offsetof(regk_dns_in, off), offsetof(regk_dns_in, k),
               offsetof(regk_dns_in, total), offsetof(regk_dns_in, flags), offsetof(regk_dns_in, reserved));
        printf("%zu %zu %zu ", sizeof(regk_dns_opts), offsetof(regk_dns_opts, udp_payload), sizeof(regk_dns_out));
        printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu ", offsetof(regk_dns_out, resp_total),
               offsetof(regk_dns_out, n_status), offsetof(regk_dns_out, n_truncated), offsetof(regk_dns_out, flags),
               offsetof(regk_dns_out, launches), offsetof(regk_dns_out, resp_off), offsetof(regk_dns_out, resp),
               offsetof(regk_dns_out, status), offsetof(regk_dns_out, tc), offsetof(regk_dns_out, node),
               offsetof(regk_dns_out, kernel_ms));
        printf("%u %u %u %u %u\n", REGK_DNS_TCP, REGK_DNS_NXDOMAIN, REGK_DNS_REFUSED, REGK_DNS_BADVERS, REGK_DNS_DROPPED);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    I, O, R = _native.CDnsIn, _native.CDnsOpts, _native.CDnsOut
    assert got == [C.sizeof(I), I.off.offset, I.k.offset, I.total.offset, I.flags.offset, I.reserved.offset,
                   C.sizeof(O), O.udp_payload.offset, C.sizeof(R), R.resp_total.offset, R.n_status.offset,
                   R.n_truncated.offset, R.flags.offset, R.launches.offset, R.resp_off.offset, R.resp.offset,
                   R.status.offset, R.tc.offset, R.node.offset, R.kernel_ms.offset, _native.FLAG_DNS_TCP,
                   _native.DNS_NXDOMAIN, _native.DNS_REFUSED, _native.DNS_BADVERS, _native.DNS_DROPPED]
    assert "regk_dns_answer" in _native.EXPORTS


@pytest.fixture(scope="module")
def emul(built):
    d = tempfile.mkdtemp(prefix="regk_dns_emul")
    exe = os.path.join(d, "dns_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "dns_emul.cpp")])

    def run(lines):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input="".join(x + "\n" for x in lines), capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        return [ln.split() for ln in p.stdout.splitlines()]
    yield run
    shutil.rmtree(d, ignore_errors=True)


def want_parse(msg):
    """the restatement's view, as the emulator prints it (an error response carries the status alone)"""
    r = du.parse(msg)
    st = r["status"]
    if st in (du.DROPPED, du.NOTIMP, du.FORMERR):
        return [st]
    labels = r["labels"]
    path = (b"/" + b"/".join(x.lower() for x in reversed(labels))).hex() if labels else "-"
    plain = int(all(c in du.PLAIN for x in labels for c in x))
    return [st, r["qend"], sum(len(x) + 1 for x in labels) + 1, len(labels), r["qtype"], r["qclass"], int(r["opt"]), r["do"],
            r["req"], plain, path]


def got_parse(g):
    st = int(g[0])
    if st in (du.DROPPED, du.NOTIMP, du.FORMERR):
        return [st]
    return [int(x) for x in g[:10]] + [g[10]]


def valid_queries():
    out = [du.query(b"b44c74d6.example.joyent.us"), du.query(b"_http._tcp.Example.Joyent.US", du.T_SRV),
           du.query(b"x.us", du.T_AAAA, opt=(1232, 0, 1)), du.query(b"", du.T_ANY), du.query(b"a*b.us", opt=(4096, 0, 0)),
           du.query(b"x.us", qclass=3, opt=(512, 0, 0)), du.query(b"x.us", opt=(600, 1, 1))]
    out.append(du.query(b"x.us", opt=(1232, 0, 0))[:-2] + b"\0\4abcd")        # OPT with 4 bytes of option data
    return out


def mutations():
    msgs = []
    for m in valid_queries():
        msgs += [m[:n] for n in range(len(m) + 1)]                             # every truncation point
        for i in range(min(len(m), 40)):                                       # header, counts, labels
            for v in {0, 1, 0x3F, 0x40, 0x80, 0xC0, 0xFF, m[i] ^ 1, m[i] ^ 0x80, m[i] ^ 0x20}:
                msgs.append(m[:i] + bytes([v]) + m[i + 1:])
        msgs += [m + b"\0", m + b"\0" * 11]                                    # trailing bytes
    for n in (62, 63, 64):                                                     # label lengths
        msgs.append(du.query(b"a" * n + b".us"))
    for total in (254, 255, 256, 257):                                         # wire names around 255 bytes
        labels, rest = [], total - 1
        while rest > 0:
            k = min(63, rest - 1)
            labels.append(b"c" * k)
            rest -= k + 1
        name = b".".join(labels)
        assert len(du.wire_name(name)) == total
        msgs.append(du.query(name))
    hdr = struct.pack(">HHHHHH", 7, 0x0100, 1, 0, 0, 0)
    msgs += [hdr + b"\x01a\xc0\x0c\0\1\0\1", hdr + b"\xc0\x0c\0\1\0\1", hdr + b"\x41a\0\0\1\0\1", hdr + b"\x81\0\0\1\0\1"]
    base = du.query(b"x.us")
    ar1 = base[:10] + b"\0\1" + base[12:]
    msgs += [ar1 + b"\0" + struct.pack(">HHIH", 41, 1232, 0, 5) + b"abcd",        # RDATA past the message
             ar1 + b"\1a\0" + struct.pack(">HHIH", 41, 1232, 0, 0),               # owner not the root
             ar1 + b"\0" + struct.pack(">HHIH", 1, 1232, 0, 0),                   # not an OPT
             ar1 + b"\0" + struct.pack(">HHIH", 41, 100, 0, 0) + b"\0",           # trailing byte
             ar1 + b"\0" + struct.pack(">HHIH", 41, 100, 0x00FF8000, 0),         # version 255, DO
             ar1, base[:10] + b"\0\2" + base[12:]]
    msgs += [bytes(range(12)), b"", b"\0" * 11, b"\0\0\x80" + b"\0" * 9]
    return msgs


def test_parser_against_the_restatement(emul):
    msgs = mutations()
    got = emul(["P " + (m.hex() or "-") for m in msgs])
    assert len(got) == len(msgs)
    statuses = set()
    for m, g in zip(msgs, got):
        w = want_parse(m)
        statuses.add(w[0])
        assert got_parse(g) == w, (m.hex(), g, w)
    assert statuses == {du.ANSWER, du.FORMERR, du.NOTIMP, du.REFUSED, du.BADVERS, du.DROPPED}


def brute_fit(kind, L, qend, opt, kids):
    """RR by RR: (nans, nadd, ans_bytes, tc, response bytes)"""
    size = qend + (11 if opt else 0)
    if kind != 3:
        rrs, extra = [16] * (1 if kind == 1 else len(kids)), []
    else:
        rrs, extra, at = [], [], qend
        for np_, ln in kids:
            if np_:
                extra.append(at + 18)
            rrs += [20 + ln] * np_
            at += np_ * (20 + ln)
    nans = 0
    for r in rrs:
        if size + r > L:
            break
        size += r
        nans += 1
    tc = int(nans < len(rrs))
    ans_bytes = size - qend - (11 if opt else 0)
    nadd = 0
    if not tc:
        for ptr in extra:
            if ptr > 0x3FFF or size + 16 > L:
                break
            size += 16
            nadd += 1
    return [nans, nadd, ans_bytes, tc, size]


def test_truncation_arithmetic(emul):
    rng = random.Random(1)
    cases = []
    for _ in range(400):
        kind = rng.choice([1, 2, 3, 3, 3])
        kids = [] if kind == 1 else [(rng.choice([0, 1, 1, 2, 5, 40]), rng.randrange(1, 254)) for _ in range(rng.randrange(0, 60))]
        qend, opt = rng.randrange(17, 272), rng.randrange(2)
        full = brute_fit(kind, 65535, qend, opt, kids)[4]
        for L in {512, 1232, 65535, full - 1, full, full + 1, rng.randrange(512, 4096)}:
            if 512 <= L <= 65535:
                cases.append((kind, L, qend, opt, kids))
    # pointers past 0x3FFF: many children, all answers fit over TCP
    cases.append((3, 65535, 40, 1, [(1, 200)] * 120 + [(0, 5)] * 3 + [(2, 30)] * 10))
    cases.append((3, 65535, 271, 0, [(1, 63)] * 196))
    lines = ["F %d %d %d %d %d %s" % (k, L, q, o, len(kids), " ".join("%d %d" % x for x in kids)) for k, L, q, o, kids in cases]
    got = emul(lines)
    seen_tc = seen_reach = 0
    for c, g in zip(cases, got):
        w = brute_fit(*c)
        assert [int(x) for x in g] == w, (c, g, w)
        seen_tc += w[3]
        seen_reach += c[1] == 65535 and not w[3] and w[1] < sum(1 for n, _ in c[4] if n)
    assert seen_tc > 50 and seen_reach >= 2


def zone_queries(zone, nodes, rng):
    """every owner asked every way, and names that own nothing"""
    msgs = []
    for j, (path, _) in enumerate(nodes):
        name = rv.name_of(path)
        for t in (du.T_A, du.T_SRV, du.T_AAAA):
            msgs.append(du.query(name, t, ident=rng.randrange(65536)))
        if j in zone.srv:
            rec = zone.rec[j]
            for t in (du.T_SRV, du.T_A, du.T_ANY):
                for opt in (None, (512, 0, 1), (4096, 0, 0), (1232, 1, 0)):
                    msgs.append(du.query(rec[1] + b"." + rec[2] + b"." + name.upper(), t, opt=opt))
    msgs += [du.query(b"nope.example"), du.query(b"a b.us"), du.query(b"", du.T_A)]
    return msgs


def rrsets(text):
    """presentation lines as dnspython RRsets, built as from_wire builds them: {(name, type): (ttl, rdataset)}"""
    import dns.message
    import dns.rdata
    import dns.rdataclass
    import dns.rdatatype
    m = dns.message.Message()
    for ln in text.decode().splitlines():
        name, ttl, _, typ, rd = ln.split("\t")
        rt = dns.rdatatype.from_text(typ)
        rs = m.find_rrset(m.answer, dns.name.from_text(name), dns.rdataclass.IN, rt, create=True)
        rs.add(dns.rdata.from_text(dns.rdataclass.IN, rt, rd), int(ttl))
    return {(rs.name, rs.rdtype): (rs.ttl, set(rs)) for rs in m.answer}


def decoded(section):
    return {(rs.name, rs.rdtype): (rs.ttl, set(rs)) for rs in section}


def check_with_dnspython(zone, msgs, udp, tcp):
    pytest.importorskip("dns")
    import dns.flags
    import dns.message
    res = zone.resolved
    by_node = {(k, j): res["sections"][q] for q, (k, j) in enumerate(zip(res["q_kind"], res["q_node"]))}
    for m in msgs:
        st, tc, node, resp = du.answer(zone, m, udp, tcp)
        if st == du.DROPPED:
            assert resp == b""
            continue
        r = dns.message.from_wire(resp)
        assert bool(r.flags & dns.flags.TC) == bool(tc)
        q = du.parse(m)
        if st != du.ANSWER:
            assert not r.answer and not tc
            continue
        if tc:
            continue
        if q["qtype"] == du.T_A:
            kind = zone.a[node][0]
            assert decoded(r.answer) == rrsets(by_node[(kind, node)][0])
            assert not [x for x in r.additional if x.rdtype != 41]
        else:
            ans, add = by_node[(rv.SERVICE_SRV, node)]
            assert decoded(r.answer) == rrsets(ans)
            got, want = decoded([x for x in r.additional if x.rdtype != 41]), rrsets(add)
            n_add = struct.unpack(">H", resp[10:12])[0] - (1 if q["opt"] else 0)
            if n_add == len(add.splitlines()):
                assert got == want
            else:
                assert all(k in want and want[k][0] == v[0] and v[1] <= want[k][1] for k, v in got.items())


@pytest.mark.parametrize("udp,tcp", [(512, False), (1232, False), (65535, True)])
def test_restatement_decodes_with_dnspython(udp, tcp):
    rng = random.Random(udp)
    scen = list(readme_scenarios().values())
    big = [(b"/us/big", service(b"_h", b"_tcp", 8080, 30))]
    big += [(b"/us/big/i%03d" % i, host(b"redis_host", b"10.0.0.%d" % (i % 250), [None, 10][i % 2],
                                       [None, [], [1, 2, 3]][i % 3])) for i in range(300)]
    for nodes in scen + [big]:
        zone = du.Zone(nodes)
        check_with_dnspython(zone, zone_queries(zone, nodes, rng), udp, tcp)


def test_restatement_worked_by_hand():
    nodes = [(b"/us/x", service(b"_a", b"_udp", 53, None)),
             (b"/us/x/h1", host(b"rr_host", b"10.0.0.1", 5, [1, 2]))]
    zone = du.Zone(nodes, 30, 60)
    st, tc, node, resp = du.answer(zone, du.query(b"_A._udp.x.US", du.T_SRV, ident=0xBEEF), 1232)
    q = b"\x02_A\x04_udp\x01x\x02US\x00\x00\x21\x00\x01"
    target = b"\x02h1\x01x\x02us\x00"
    srv = lambda port: b"\xc0\x0c\x00\x21\x00\x01" + struct.pack(">IH", 60, 6 + len(target)) + struct.pack(">HHH", 0, 10, port) + target
    add = struct.pack(">H", 0xC000 | (12 + len(q) + 18)) + b"\x00\x01\x00\x01" + struct.pack(">IH", 5, 4) + bytes([10, 0, 0, 1])
    assert (st, tc, node) == (du.ANSWER, 0, 0)
    assert resp == b"\xbe\xef\x85\x00\x00\x01\x00\x02\x00\x00\x00\x01" + q + srv(1) + srv(2) + add
