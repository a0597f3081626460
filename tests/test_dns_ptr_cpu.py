"""regk_dns_answer with REGK_DNS_PTR on the CPU: the restatement in dns_ptr_util on hand-built cases (the README's
three names on one address, queryable and non-queryable types, node classes, NODATA on a PTR owner), the
reverse-name recogniser and the PTR truncation cut of regk_dns_ptr.cuh compiled with g++ under AddressSanitizer
against the restatement, and the flag's value in the header."""
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import dns_ptr_util as pu
import dns_util as du
from test_resolve_cpu import alias_node, host, readme_scenarios, service

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
README_ADDR = b"172.27.10.72"


def rr_list(resp, qend, n):
    """(ttl, target name) of n PTR RRs after the question"""
    out, i = [], qend
    for _ in range(n):
        owner, typ, cls, ttl, rdlen = struct.unpack(">HHHIH", resp[i:i + 12])
        assert (owner, typ, cls) == (0xC00C, pu.T_PTR, 1)
        w = resp[i + 12:i + 12 + rdlen]
        labels, k = [], 0
        while w[k]:
            labels.append(w[k + 1:k + 1 + w[k]])
            k += w[k] + 1
        assert k + 1 == rdlen
        out.append((ttl, b".".join(labels)))
        i += 12 + rdlen
    assert i == len(resp) or resp[i] == 0                      # the OPT record, when there is one, follows
    return out


def test_readme_names_on_one_address():
    nodes = readme_scenarios()["plain"]
    zone = du.Zone(nodes)
    q = du.query(pu.reverse_name(README_ADDR), pu.T_PTR)
    st, tc, node, resp = pu.answer(zone, q)
    assert (st, tc, node) == (du.ANSWER, 0, 0)
    assert struct.unpack(">HHHHHH", resp[:12])[1:] == (0x8500, 1, 3, 0, 0)
    names = [b"b44c74d6.example.joyent.us", b"host-1a.example.joyent.us", b"host-1b.example.joyent.us"]
    assert rr_list(resp, len(q), 3) == [(30, n) for n in names]
    with_ttl = list(nodes)
    with_ttl[1] = alias_node(names[1], b"load_balancer", README_ADDR, 5)
    st, _, _, resp = pu.answer(du.Zone(with_ttl), q)
    assert rr_list(resp, len(q), 3) == [(30, names[0]), (5, names[1]), (30, names[2])]
    assert pu.answer(zone, q, ptr=False) == du.answer(zone, q)
    assert pu.answer(zone, q)[0] != du.answer(zone, q)[0]


def test_only_queryable_ok_hosts_are_targets():
    a = b"10.9.8.7"
    nodes = [(b"/us/x", service()), (b"/us/x/ops", host(b"ops_host", a)), (b"/us/x/rr", host(b"rr_host", a)),
             (b"/us/x/redis", host(b"redis_host", a, 7)), (b"/us/bad", host(b"host", a, -1)),
             (b"/us/typo", host(b"hostx", a)), (b"/us/h", host(b"host", a, 9)), (b"/us/other", host(b"host", b"10.9.8.6"))]
    zone = du.Zone(nodes)
    q = du.query(pu.reverse_name(a), pu.T_PTR, opt=(1232, 0, 1))
    st, tc, node, resp = pu.answer(zone, q)
    assert (st, tc, node) == (du.ANSWER, 0, 3)
    assert rr_list(resp, len(q) - 11, 2) == [(7, b"redis.x.us"), (9, b"h.us")]
    only_rr = [(b"/us/x", service()), (b"/us/x/rr", host(b"rr_host", a))]
    assert pu.answer(du.Zone(only_rr), q)[0] == du.NXDOMAIN


def test_nodata_on_a_ptr_owner_and_nxdomain_elsewhere():
    zone = du.Zone(readme_scenarios()["plain"])
    name = pu.reverse_name(README_ADDR)
    for qtype in (du.T_A, du.T_ANY, du.T_SRV, du.T_AAAA):
        st, tc, node, resp = pu.answer(zone, du.query(name, qtype))
        assert (st, tc, node) == (du.NODATA, 0, du.NONE)
        assert struct.unpack(">HHHHHH", resp[:12])[1:] == (0x8500, 1, 0, 0, 0)
    for other in (b"72.10.27.171.in-addr.arpa", b"10.27.172.in-addr.arpa", b"072.10.27.172.in-addr.arpa"):
        assert pu.answer(zone, du.query(other, pu.T_PTR))[0] == du.NXDOMAIN
    assert pu.answer(zone, du.query(name.upper(), pu.T_PTR))[0] == du.ANSWER


def test_a_reverse_named_host_owns_a_as_before():
    """a node whose name is itself a reverse name keeps its A answer; PTR and A are asked of one name"""
    nodes = [(b"/arpa/in-addr/1/2/3/4", host(b"host", b"1.2.3.4")), (b"/us/h", host(b"host", b"1.2.3.4"))]
    zone = du.Zone(nodes)
    name = b"4.3.2.1.in-addr.arpa"
    assert pu.answer(zone, du.query(name, du.T_A)) == du.answer(zone, du.query(name, du.T_A))
    st, _, node, resp = pu.answer(zone, du.query(name, pu.T_PTR))
    assert (st, node) == (du.ANSWER, 0)
    assert rr_list(resp, len(du.query(name, pu.T_PTR)), 2) == [(30, name), (30, b"h.us")]
    assert pu.answer(zone, du.query(name, du.T_ANY))[0] == du.NODATA


def test_cut_on_whole_rrs():
    nodes = [(b"/us/h%04d" % i, host(b"host", b"10.0.0.1")) for i in range(100)]
    zone = du.Zone(nodes)
    q = du.query(pu.reverse_name(b"10.0.0.1"), pu.T_PTR)
    st, tc, node, resp = pu.answer(zone, q)
    rr = 14 + len(b"h0000.us")
    assert (st, tc, node) == (du.ANSWER, 1, 0)
    assert len(resp) == len(q) + (512 - len(q)) // rr * rr
    assert pu.answer(zone, q, tcp=True)[1] == 0


@pytest.fixture(scope="module")
def emul(built):
    d = tempfile.mkdtemp(prefix="regk_dns_ptr_emul")
    exe = os.path.join(d, "dns_ptr_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "dns_ptr_emul.cpp")])

    def run(lines):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input="".join(x + "\n" for x in lines), capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        return [ln.split() for ln in p.stdout.splitlines()]
    yield run
    shutil.rmtree(d, ignore_errors=True)


def want_reverse(msg):
    r = du.parse(msg)
    a = pu.reverse_addr(r["labels"]) if r["status"] == du.ANSWER else None
    if a is None:
        return [str(r["status"]), "-"]
    o = [int(x) for x in a.split(b".")]
    return [str(r["status"]), str(o[0] << 24 | o[1] << 16 | o[2] << 8 | o[3])]


def octet_forms():
    """every octet label of 1-4 bytes over digits, plus a few non-digit bytes"""
    digits = [str(i).encode() for i in range(10)]
    out = list(digits)
    for n in (2, 3):
        out += [a + b for a in digits for b in digits] if n == 2 else [b"%03d" % i for i in range(1000)]
    out += [b"1000", b"2550", b"0255", b"9999", b"a", b"1a", b"-1", b"1 ", b"\xb2", b"12\x00"]
    return out


def test_recogniser_against_the_restatement(emul):
    rng = random.Random(3)
    msgs = []
    for o in octet_forms():
        for pos in range(4):
            labs = [b"1", b"2", b"3", b"4"]
            labs[pos] = o
            msgs.append(du.query(b".".join(labs) + b".in-addr.arpa", pu.T_PTR))
    for ia in (b"in-addr", b"IN-ADDR", b"In-AdDr", b"in_addr", b"inaddr", b"in-addr1"):
        for arpa in (b"arpa", b"ARPA", b"aRpA", b"arp", b"arpa1"):
            msgs.append(du.query(b"4.3.2.1." + ia + b"." + arpa, pu.T_PTR, opt=(1232, 0, 0)))
    for n in range(1, 9):                                      # 1-8 labels, the 5/6/7-label names among them
        msgs.append(du.query(b".".join(([b"1"] * (n - 2) + [b"in-addr", b"arpa"])[-n:]), pu.T_PTR))
        msgs.append(du.query(b".".join([b"7"] * n) + b".in-addr.arpa", pu.T_PTR))
    msgs += [du.query(b"255.255.255.255.in-addr.arpa", pu.T_PTR), du.query(b"0.0.0.0.in-addr.arpa", du.T_A),
             du.query(b"1.2.3.4.in-addr.arpa", pu.T_PTR, qclass=3), du.query(b"1.2.3.4.in-addr.arpa", opt=(512, 1, 0))]
    for _ in range(3000):
        labs = [bytes(rng.randrange(256) if rng.random() < 0.2 else rng.choice(b"0123456789")
                      for _ in range(rng.randrange(1, 5))) for _ in range(4)]
        tail = rng.choice([b"in-addr.arpa", b"IN-addr.Arpa", b"in-addr.arpb", b"x.arpa"])
        m = du.query(b".".join(labs) + b"." + tail, rng.choice([pu.T_PTR, du.T_A]))
        if rng.random() < 0.2:
            i = rng.randrange(len(m))
            m = m[:i] + bytes([rng.randrange(256)]) + m[i + 1:]
        msgs.append(m)
    got = emul(["R " + (m.hex() or "-") for m in msgs])
    assert [want_reverse(m) for m in msgs] == got
    assert sum(g[1] != "-" for g in got) > 500


def brute_cut(room, lens):
    size, n = 0, 0
    for x in lens:
        if size + 14 + x > room:
            break
        size += 14 + x
        n += 1
    return [str(n), str(size), str(int(n < len(lens)))]


def test_ptr_cut_against_brute_force(emul):
    rng = random.Random(5)
    cases = [(0, []), (13, [1]), (14, [0]), (15, [1]), (16, [1])]
    for _ in range(2000):
        lens = [rng.randrange(3, 254) for _ in range(rng.randrange(0, 40))]
        total = sum(14 + x for x in lens)
        cases.append((rng.choice([rng.randrange(0, total + 2), total, max(total - 1, 0), total + 1]), lens))
    got = emul(["C %d %d %s" % (room, len(lens), " ".join(map(str, lens))) for room, lens in cases])
    assert got == [brute_cut(room, lens) for room, lens in cases]


def test_flag_matches_header(built):
    from registrar_b200 import _native
    src = '#include <stdio.h>\n#include "regk.h"\nint main(void) { printf("%u %u\\n", REGK_DNS_PTR, REGK_DNS_TCP); return 0; }\n'
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    assert got == [_native.FLAG_DNS_PTR, _native.FLAG_DNS_TCP]
    assert _native.FLAG_DNS_PTR & (_native.FLAG_OUT_DEVICE | _native.FLAG_DNS_TCP) == 0
