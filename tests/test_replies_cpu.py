"""regk_read_replies on the CPU: the restatement in replies_util against frames worked out by hand from zookeeper.jute,
and the per-frame helpers of regk_replies.cuh (reply_head, reply_check), compiled with g++ under AddressSanitizer,
against the restatement's sequential reader on every truncation point of a small stream, random byte streams, and
streams whose node data embeds well-formed fake reply frames."""
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import reconcile_owned_util as ou
import replies_util as ru

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SESSION, OTHER = 0x1234_5678_9ABC_DEF0, 0x0FED_CBA9_8765_4321

# GetDataRequest{"/a", watch = false}, xid 5, worked out by hand
ONE_GETDATA = bytes.fromhex("0000000f" "00000005" "00000004" "00000002" "2f61" "00")

# GetDataResponse to it: data "x", Stat{czxid 2^32, mzxid 2^32 + 5, ctime, mtime, version 7, cversion 3, aversion 0,
# ephemeralOwner 0x0123456789abcdef, dataLength 1, numChildren 2, pzxid 2^32 + 9}, zxid 2^33, worked out by hand
ONE_REPLY = bytes.fromhex(
    "00000059" "00000005" "0000000200000000" "00000000"                       # len 89, ReplyHeader{5, zxid, err 0}
    "00000001" "78"                                                           # data "x"
    "0000000100000000" "0000000100000005" "0000018bcfe56800" "0000018bcfe569f4"   # czxid mzxid ctime mtime
    "00000007" "00000003" "00000000" "0123456789abcdef"                       # version cversion aversion ephemeralOwner
    "00000001" "00000002" "0000000100000009")                                 # dataLength numChildren pzxid


def test_builders_worked_out_by_hand():
    assert ru.getdata_frames([b"/a"], 5) == ONE_GETDATA
    assert ru.parse_getdata(ONE_GETDATA + ru.getdata_frames([b"/bc"], -1)) == [(5, b"/a"), (-1, b"/bc")]
    assert len(ONE_REPLY) == 4 + 88 + 1
    assert ru.success(5, b"x", 7, 0x0123456789ABCDEF, 2, seed=0) == ONE_REPLY
    assert ru.error(5, ru.NONODE) == bytes.fromhex("00000010" "00000005" "0000000000000007" "ffffff9b")
    assert ru.ping() == bytes.fromhex("00000010" "fffffffe" "ffffffffffffffff" "00000000")
    null = ru.success(9, b"", seed=0, null=True)
    assert len(null) == 92 and null[20:24] == b"\xff\xff\xff\xff" and null[76:80] == b"\0\0\0\0"
    r = ru.read(ONE_REPLY, 5, 1)
    assert r["found"] == [(0, b"x", 7, 0x0123456789ABCDEF)] and r["consumed"] == len(ONE_REPLY)


def test_reply_builder_answers_the_model():
    zk = ou.ZooKeeper()
    assert zk.create(b"/a", b"", 0, ephemeral=False) == ou.ZOK
    assert zk.create(b"/a/b", b"data", SESSION) == ou.ZOK
    assert zk.set_data(b"/a/b", b"more") == ou.ZOK
    frames = ru.getdata_frames([b"/a/b", b"/a/c", b"/a", b"/a/b"], 2 ** 31 - 2)
    s = ru.replies(zk, frames, errors={3: -4}, extra={0: ru.ping(), 2: ru.notification(b"/a"), 4: ru.ping()},
                   trailing=b"\0\0")
    r = ru.read(s, 2 ** 31 - 2, 4)
    assert r["err"] == [0, ru.NONODE, 0, -4] and r["n_skipped"] == 2
    assert r["found"] == [(0, b"more", 1, SESSION), (2, b"", 0, 0)]
    assert r["consumed"] == len(s) - 2 - len(ru.ping())
    rec, nodes = ru.snapshot_nodes([b"/a/b", b"/a/c", b"/a", b"/a/b"], r)
    assert rec == [0, 2] and nodes[0] == (b"/a/b", b"more", 1, SESSION)
    with pytest.raises(ru.Refused) as e:
        ru.read(s[:-(2 + len(ru.ping()) + 3)], 2 ** 31 - 2, 4)
    assert (e.value.code, e.value.k) == (ru.TRUNC, 3)


@pytest.fixture(scope="module")
def emul(built):
    d = tempfile.mkdtemp(prefix="regk_replies_emul")
    exe = os.path.join(d, "replies_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "replies_emul.cpp")])

    def run(cases):
        """cases = [(stream, xid_base, n)] -> [(plausibility codes, read result)]"""
        lines = []
        for b, xb, n in cases:
            lines += ["S %s %d %d" % (b.hex() or "-", xb, n), "P", "R"]
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        out = p.stdout.split("\n")
        return [([int(x) for x in out[2 * i].split()], [int(x) for x in out[2 * i + 1].split()]) for i in range(len(cases))]
    yield run
    shutil.rmtree(d, ignore_errors=True)


def want(b, xb, n):
    codes = [ru.plausible(b, pos, xb, n) for pos in range(len(b))]
    try:
        r = ru.read(b, xb, n)
        return codes, [0, r["consumed"], r["n_skipped"]] + r["err"]
    except ru.Refused as e:
        return codes, [e.code, e.pos, e.k]


def small_stream(xb=7):
    zk = ou.ZooKeeper()
    zk.create(b"/r", b"", 0, ephemeral=False)
    for k in range(4):
        zk.create(b"/r/n%d" % k, b"v" * k, SESSION if k % 2 else OTHER)
    paths = [b"/r/n0", b"/r/n1", b"/r/zz", b"/r/n3", b"/r/n2"]
    return ru.replies(zk, ru.getdata_frames(paths, xb), errors={3: -102}, null={0},
                      extra={1: ru.ping(), 3: ru.notification(b"/r/n1"), 5: ru.ping()}), len(paths)


def test_every_truncation_point(emul):
    b, n = small_stream()
    cases = [(b[:t], 7, n) for t in range(len(b) + 1)]
    got = emul(cases)
    for (s, xb, nn), g in zip(cases, got):
        assert g == want(s, xb, nn), len(s)
    assert got[-1][1][:3] == [0, len(b) - len(ru.ping()), 2]


def test_random_byte_streams(emul):
    rng = random.Random(5)
    cases = []
    for trial in range(300):
        ln = rng.randrange(0, 200)
        b = bytearray(rng.getrandbits(8) for _ in range(ln))
        xb = rng.choice([0, 1, 2 ** 31 - 2, -2 ** 31, 1000])
        n = rng.randrange(1, 6)
        if ln >= 24 and trial % 2:                  # plant plausible heads: small lengths, in-range xids
            for _ in range(3):
                p = rng.randrange(0, ln - 23)
                b[p:p + 4] = struct.pack(">i", rng.choice([16, 20, 88, 89, ln - p - 4, rng.randrange(-5, 120)]))
                b[p + 4:p + 8] = struct.pack(">i", rng.choice([ru.wrap(xb + rng.randrange(n)), -1, -2, -3]))
                b[p + 16:p + 20] = struct.pack(">i", rng.choice([0, 0, ru.NONODE]))
                b[p + 20:p + 24] = struct.pack(">i", rng.choice([-2, -1, 0, 1, ln]))
        cases.append((bytes(b), xb, n))
    for (s, xb, n), g in zip(cases, emul(cases)):
        assert g == want(s, xb, n), (s.hex(), xb, n)


def test_data_embedding_fake_frames(emul):
    """node data that holds well-formed reply frames with the right xids: the reader follows the lengths, not them"""
    xb, n = 100, 6
    fakes = b"".join(ru.success(ru.wrap(xb + k), b"fake%d" % k, 9, OTHER, seed=k) for k in range(n)) + ru.ping()
    zk = ou.ZooKeeper()
    paths = [b"/f%d" % k for k in range(n)]
    for k, p in enumerate(paths):
        zk.create(p, fakes[k:] + fakes[:k], SESSION)
    b = ru.replies(zk, ru.getdata_frames(paths, xb), extra={2: ru.notification(fakes)})
    cases = [(b, xb, n), (b[:len(b) - 3], xb, n), (b[:300], xb, n)]
    got = emul(cases)
    for (s, x, nn), g in zip(cases, got):
        assert g == want(s, x, nn)
    assert got[0][1][:3] == [0, len(b), 1]
    assert sum(1 for c in got[0][0] if c == ru.OK) > n + 1 + n      # the planted frames are plausible positions too
