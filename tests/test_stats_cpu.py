"""The heartbeat by stat on the CPU: the restatement in stats_util against an ExistsRequest and an ExistsResponse worked
out by hand from zookeeper.jute; the struct layouts against the C compiler; and the helpers of regk_stats.cuh (stat_head,
stat_check, and stat_mask16, the candidate test from registers), compiled with g++ under AddressSanitizer, against the
restatement: every position's verdict and a front-to-back read over every truncation point of a small stream, random
streams with planted heads, and streams whose notification paths embed well-formed stat replies with in-range xids."""
import ctypes as C
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import reconcile_owned_util as ou
import stats_util as su

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# ExistsRequest{"/a", watch = false} with xid 5: len = 4 + 4 + (4 + 2) + 1 = 15
ONE_REQUEST = bytes.fromhex("0000000f" "00000005" "00000003" "00000002" "2f61" "00")

# ExistsResponse to xid 6, zxid 2^33 + 2^32: Stat{czxid 2^32, mzxid 2^32 + 5, ctime 1.7e12 ms, mtime + 500, version 1,
# cversion 3, aversion 0, ephemeralOwner 0x1234567800000009, dataLength 3, numChildren 0, pzxid 2^32 + 9}: len = 16 + 68
ONE_REPLY = bytes.fromhex(
    "00000054" "00000006" "0000000300000000" "00000000"
    "0000000100000000" "0000000100000005" "0000018bcfe56800" "0000018bcfe569f4"
    "00000001" "00000003" "00000000" "1234567800000009" "00000003" "00000000" "0000000100000009")


def test_frames_worked_out_by_hand():
    assert su.exists_frames([b"/a"], 5) == ONE_REQUEST
    assert su.parse_exists(ONE_REQUEST) == [(5, b"/a")]
    assert su.success(6, version=1, owner=0x1234567800000009, data_len=3, zxid=0x300000000) == ONE_REPLY
    # the fields regk_read_stats takes, at their byte positions
    assert len(ONE_REPLY) == 88
    assert ONE_REPLY[28:36] == struct.pack(">q", 2 ** 32 + 5)                       # mzxid
    assert ONE_REPLY[52:56] == struct.pack(">i", 1)                                 # version
    assert ONE_REPLY[64:72] == struct.pack(">q", 0x1234567800000009)                # ephemeralOwner
    assert ONE_REPLY[72:76] == struct.pack(">i", 3)                                 # dataLength
    r = su.read(ONE_REPLY, 6, 1)
    assert (r["err"], r["version"], r["owner"], r["data_length"], r["mzxid"]) == ([0], [1], [0x1234567800000009], [3],
                                                                                  [2 ** 32 + 5])
    assert r["consumed"] == 88
    r = su.read(su.ping() + su.error(9, su.NONODE) + b"tail", 9, 1)
    assert r["err"] == [su.NONODE] and r["n_missing"] == 1 and r["n_skipped"] == 1 and r["consumed"] == 40
    # the classification table
    paths, pays = [b"/p", b"/q", b"/p", b"/r", b"/s"], [b"abc", b"abc", b"abc", b"abc", b"abc"]
    s = b"".join([su.success(1, 4, 7, 3, seed=1), su.error(2, su.NONODE), su.success(3, 4, 7, 3, seed=1),
                  su.success(4, 2, 8, 3, seed=2), su.success(5, 9, 7, 4, seed=3)])
    r = su.read(s, 1, 5)
    c = su.classify(paths, pays, r, 7, 1)
    assert c["cls"] == [su.SAME, su.CREATE, su.DUP, su.REPLACE, su.UPDATE] and c["match"] == [0, su.NO_MATCH, 0, 3, 4]
    assert c["update_ver"] == [9] and c["replace_ver"] == [2]
    known = list(r["mzxid"])
    known[0] += 1
    assert su.classify(paths, pays, r, 7, 1, known)["cls"][0] == su.UPDATE
    assert su.classify(paths, pays, r, 7, 0)["cls"][0] == su.REPLACE                 # persistent wanted, ephemeral found


def test_struct_layouts_match_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu ", sizeof(regk_stats), offsetof(regk_stats, n_found),
               offsetof(regk_stats, consumed), offsetof(regk_stats, flags), offsetof(regk_stats, launches),
               offsetof(regk_stats, err), offsetof(regk_stats, version), offsetof(regk_stats, ephemeral_owner),
               offsetof(regk_stats, data_length), offsetof(regk_stats, mzxid));
        printf("%zu %zu %zu %zu %zu %u\n", offsetof(regk_stats, kernel_ms), sizeof(regk_stat_opts),
               offsetof(regk_stat_opts, zk_flags), offsetof(regk_stat_opts, reserved), offsetof(regk_stat_opts, known_mzxid),
               REGK_ZK_EXISTS);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    S, O = _native.CStats, _native.CStatOpts
    assert got == [C.sizeof(S), S.n_found.offset, S.consumed.offset, S.flags.offset, S.launches.offset, S.err.offset,
                   S.version.offset, S.ephemeral_owner.offset, S.data_length.offset, S.mzxid.offset, S.kernel_ms.offset,
                   C.sizeof(O), O.zk_flags.offset, O.reserved.offset, O.known_mzxid.offset, _native.ZK_EXISTS]
    assert "regk_read_stats" in _native.EXPORTS and "regk_reconcile_stats" in _native.EXPORTS


@pytest.fixture(scope="module")
def emul(built):
    d = tempfile.mkdtemp(prefix="regk_stats_emul")
    exe = os.path.join(d, "stats_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "stats_emul.cpp")])

    def run(cases):
        """cases = [(stream, xid_base, n, start)] -> [(head codes, mask bits, read result)]"""
        lines = []
        for b, xb, n, start in cases:
            lines += ["S %s" % (b.hex() or "-"), "X %d %d" % (xb, n), "P", "M %d" % start, "R %d" % start]
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        out = p.stdout.split("\n")
        return [([int(x) for x in out[3 * i].split()], [int(x) for x in out[3 * i + 1].split()], out[3 * i + 2].split())
                for i in range(len(cases))]
    yield run
    shutil.rmtree(d, ignore_errors=True)


def want(b, xb, n, start=0):
    codes = [su.plausible(b, pos, xb, n) for pos in range(len(b))]
    mask = [int(c == su.OK and pos >= start) for pos, c in enumerate(codes)]
    try:
        r = su.read(b, xb, n, start)
        recs = sum(([str(v) for v in t] for t in zip(r["err"], r["version"], r["owner"], r["data_length"], r["mzxid"])), [])
        return codes, mask, ["0", str(r["consumed"]), str(r["n_skipped"])] + recs
    except su.Refused as e:
        return codes, mask, [str(e.code), str(e.pos), str(e.k)]


def check(emul, cases):
    for c, g in zip(cases, emul(cases)):
        assert g == want(*c), (c[0].hex(), c[1:])


def scenario(xb=7, seed=1):
    """eight exists frames answered by the model: found (several owners, versions, lengths), missing, another error;
    a ping and a notification between the replies"""
    rng = random.Random(seed)
    zk = ou.ZooKeeper()
    zk.create(b"/d", b"", 0, ephemeral=False)
    paths = [b"/d/n%d" % i for i in range(8)]
    for i, p in enumerate(paths):
        if i % 3 != 1:
            zk.create(p, b"x" * rng.randrange(0, 40), rng.choice([0, 5, 2 ** 62 + 3]), ephemeral=i % 2 == 0)
            for _ in range(rng.randrange(3)):
                zk.set_data(p, b"y" * rng.randrange(0, 9))
    fb = su.exists_frames(paths, xb)
    return su.replies(zk, fb, errors={5: -4}, extra={0: su.ping(), 2: su.notification(b"/d")}), len(paths)


def test_every_truncation_point_and_start_phase(emul):
    s, n = scenario()
    assert su.read(s, 7, n)["n_found"] and su.read(s, 7, n)["n_missing"] and su.read(s, 7, n)["n_error"] == 1
    cases = [(s[:t], 7, n, 0) for t in range(len(s) + 1)]
    for phase in range(17):
        cases.append((bytes(range(1, phase + 1)) + s + b"\x00\x00", 7, n, phase))
    for xb in (2 ** 31 - 4, -2 ** 31, 0):                                              # xids that wrap
        cases.append((scenario(xb)[0], xb, n, 0))
    check(emul, cases)


def test_random_streams_with_planted_heads(emul):
    rng = random.Random(5)
    cases = []
    for trial in range(400):
        xb = rng.choice([0, 1, 2 ** 31 - 2, -2 ** 31, 1000])
        n = rng.choice([1, 3, 8, 2 ** 31])
        ln = rng.randrange(0, 260)
        b = bytearray(rng.getrandbits(8) for _ in range(ln))
        if ln >= 24 and trial % 2:
            for _ in range(4):
                p = rng.randrange(0, ln - 19)
                b[p:p + 4] = struct.pack(">i", rng.choice([16, 84, 84, ln - p - 4, 15, rng.randrange(-5, 200)]))
                b[p + 4:p + 8] = struct.pack(">i", rng.choice([su.wrap(xb + rng.randrange(min(n, 9))), -1, -2, -3, su.wrap(xb + n)]))
                b[p + 16:p + 20] = struct.pack(">i", rng.choice([0, 0, su.NONODE]))
        cases.append((bytes(b), xb, n, min(rng.choice([0, 0, 1, 5, 16, 17]), ln)))
    # well-formed streams with one byte changed
    for _ in range(300):
        base, n = scenario(seed=rng.randrange(4))
        b = bytearray(base)
        b[rng.randrange(len(b))] = rng.choice([0, 1, 0xFF, 0xFE, 0x80, rng.getrandbits(8)])
        cases.append((bytes(b), 7, n, 0))
    # a reply out of order, a reply twice, a negative Stat.dataLength
    cases.append((su.error(7, su.NONODE) + su.success(9, 1, 0, 2) + su.error(8, su.NONODE), 7, 3, 0))
    cases.append((su.error(7, su.NONODE) + su.error(7, su.NONODE), 7, 3, 0))
    cases.append((su.error(7, -4) + su.success(8, 1, 0, -1) + su.error(9, su.NONODE), 7, 3, 0))
    check(emul, cases)
    assert {want(*c)[2][0] for c in cases} >= {str(k) for k in (su.OK, su.TRUNC, su.BAD_LEN, su.NEG_XID, su.XID_RANGE,
                                                               su.ERR_BODY, su.SUCC_LEN, su.ORDER, su.NEG_DLEN)}


def test_notification_paths_that_embed_stat_replies(emul):
    """a watch notification whose path holds complete, well-formed stat replies to xids of the framing: every position
    inside it is plausible on its own, and the front-to-back read steps over the whole notification"""
    s, n = scenario()
    inner = su.success(8, 3, 0, 5, seed=9) + su.error(9, su.NONODE) + su.success(10, 1, 0, 2, seed=4)
    cases = []
    for at in (0, 3, n):
        for phase in (0, 1, 7, 15):
            zk = ou.ZooKeeper()
            paths = [b"/e/n%d" % i for i in range(n)]
            st = su.replies(zk, su.exists_frames(paths, 7), extra={at: su.notification(b"/" + inner)})
            cases.append((b"\x00" * phase + st, 7, n, phase))
    check(emul, cases)
    codes = want(*cases[0])[0]
    assert sum(c == su.OK for c in codes) > n + 1                                     # the embedded heads are plausible
