"""regk_read_children on the CPU: the restatement in children_util against a request and a response worked out by hand
from zookeeper.jute, and the per-frame helpers of regk_children.cuh (children_head, children_check, children_entry),
compiled with g++ under AddressSanitizer, against the restatement's sequential reader: every truncation point of a small
stream, random streams with planted heads, names of every length 1..300 at every byte phase, names whose bytes look like
length words, counts -1 / 0, and counts too large for their frame."""
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import children_util as cu
import reconcile_owned_util as ou

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# GetChildrenRequest{"/a", watch = false}, xid 5, worked out by hand
ONE_REQUEST = bytes.fromhex("0000000f" "00000005" "00000008" "00000002" "2f61" "00")

# GetChildrenResponse to it: children "h1" and "web", zxid 2^33, worked out by hand: len = 16 + 4 + (4 + 2) + (4 + 3) = 33
ONE_RESPONSE = bytes.fromhex(
    "00000021" "00000005" "0000000200000000" "00000000"          # len 33, ReplyHeader{5, zxid, err 0}
    "00000002"                                                   # count 2
    "00000002" "6831"                                            # "h1"
    "00000003" "776562")                                         # "web"


def test_builders_worked_out_by_hand():
    assert cu.getchildren_frames([b"/a"], 5) == ONE_REQUEST
    assert cu.parse_getchildren(ONE_REQUEST + cu.getchildren_frames([b"/bc"], -1)) == [(5, b"/a"), (-1, b"/bc")]
    assert cu.success(5, [b"h1", b"web"]) == ONE_RESPONSE
    assert cu.null_vector(5) == bytes.fromhex("00000014" "00000005" "0000000200000000" "00000000" "ffffffff")
    assert cu.error(5, cu.NONODE) == bytes.fromhex("00000010" "00000005" "0000000000000007" "ffffff9b")
    r = cu.read(ONE_RESPONSE, 5, 1)
    assert r["names"] == [[b"h1", b"web"]] and r["consumed"] == len(ONE_RESPONSE)


def test_reply_builder_answers_the_model():
    zk = ou.ZooKeeper()
    for p in (b"/a", b"/a/b", b"/a/c", b"/a/b/x", b"/e"):
        assert zk.create(p, b"", 0, ephemeral=False) == ou.ZOK
    dirs = [b"/a", b"/z", b"/e", b"/a/b", b"/a"]
    s = cu.replies(zk, cu.getchildren_frames(dirs, 2 ** 31 - 2), errors={4: -4}, null={2},
                   extra={0: cu.ping(), 2: cu.notification(b"/a"), 5: cu.ping()}, trailing=b"\0\0")
    r = cu.read(s, 2 ** 31 - 2, 5)
    assert r["err"] == [0, cu.NONODE, 0, 0, -4] and r["n_skipped"] == 2
    assert r["names"] == [[b"b", b"c"], [], [], [b"x"], []]
    assert r["consumed"] == len(s) - 2 - len(cu.ping())
    with pytest.raises(cu.Refused) as e:
        cu.read(s[:-(2 + len(cu.ping()) + 3)], 2 ** 31 - 2, 5)
    assert (e.value.code, e.value.k) == (cu.TRUNC, 4)


def test_dir_set_and_keep_rule():
    paths = [b"/c/b/a/h1", b"/c/b/a/x/y/h2", b"/top", b"/c/b/a/h3", b"/c/b//a/h4", b"/c/b/a/x/y/h5"]
    listed, unlisted = cu.dir_set(paths)
    assert listed == [(0, b"/c/b/a"), (1, b"/c/b/a/x/y")] and unlisted == [2, 4]
    r = dict(names=[[b"h1", b"x", b"h9", b"h3"], [b"h2", b"old"]])
    listing, off, cls, stale = cu.classify(paths, r)
    assert off == [0, 4, 6]
    assert listing[1] == b"/c/b/a/x" and cls == [cu.KEEP, cu.KEEP, cu.STALE, cu.KEEP, cu.KEEP, cu.STALE]
    assert stale == [2, 5]


@pytest.fixture(scope="module")
def emul(built):
    d = tempfile.mkdtemp(prefix="regk_children_emul")
    exe = os.path.join(d, "children_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "children_emul.cpp")])

    def run(cases):
        """cases = [(stream, xid_base, d, start)] -> [(plausibility codes, read result)]"""
        lines = []
        for b, xb, d, start in cases:
            lines += ["S %s %d %d" % (b.hex() or "-", xb, d), "P", "R %d" % start]
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        out = p.stdout.split("\n")
        return [([int(x) for x in out[2 * i].split()], [int(x) for x in out[2 * i + 1].split()]) for i in range(len(cases))]
    yield run
    shutil.rmtree(d, ignore_errors=True)


def want(b, xb, d, start=0):
    codes = [cu.plausible(b, pos, xb, d) for pos in range(len(b))]
    try:
        r = cu.read(b, xb, d, start)
        return codes, [0, r["consumed"], r["n_skipped"], sum(len(n) for n in r["names"])] + r["err"]
    except cu.Refused as e:
        return codes, [e.code, e.pos, e.k]


def check(emul, cases):
    for (s, xb, d, start), g in zip(cases, emul(cases)):
        assert g == want(s, xb, d, start), (s.hex(), xb, d, start)


def small_stream(xb=7):
    zk = ou.ZooKeeper()
    for p in (b"/r", b"/r/n0", b"/r/n1", b"/r/n1/q", b"/s"):
        zk.create(p, b"", 0, ephemeral=False)
    dirs = [b"/r", b"/s", b"/zz", b"/r/n1", b"/r"]
    return cu.replies(zk, cu.getchildren_frames(dirs, xb), errors={4: -102}, null={1},
                      extra={1: cu.ping(), 3: cu.notification(b"/r/n1"), 5: cu.ping()}), len(dirs)


def test_every_truncation_point(emul):
    b, d = small_stream()
    cases = [(b[:t], 7, d, 0) for t in range(len(b) + 1)]
    check(emul, cases)
    assert emul(cases[-1:])[0][1][:4] == [0, len(b) - len(cu.ping()), 2, 3]


def test_random_streams_with_planted_heads(emul):
    rng = random.Random(5)
    cases = []
    for trial in range(300):
        ln = rng.randrange(0, 200)
        b = bytearray(rng.getrandbits(8) for _ in range(ln))
        xb = rng.choice([0, 1, 2 ** 31 - 2, -2 ** 31, 1000])
        d = rng.randrange(1, 6)
        if ln >= 24 and trial % 2:
            for _ in range(3):
                p = rng.randrange(0, ln - 23)
                b[p:p + 4] = struct.pack(">i", rng.choice([16, 20, 25, ln - p - 4, rng.randrange(-5, 120)]))
                b[p + 4:p + 8] = struct.pack(">i", rng.choice([cu.wrap(xb + rng.randrange(d)), -1, -2, -3]))
                b[p + 16:p + 20] = struct.pack(">i", rng.choice([0, 0, cu.NONODE]))
                b[p + 20:p + 24] = struct.pack(">i", rng.choice([-2, -1, 0, 1, 2, ln]))
        cases.append((bytes(b), xb, d, min(rng.choice([0, 0, 1, 5]), ln)))
    # well-formed streams with one byte changed
    base, d = small_stream(11)
    for _ in range(200):
        b = bytearray(base)
        b[rng.randrange(len(b))] = rng.choice([0, 0x2F, 0x2E, 0xFF, 1, rng.getrandbits(8)])
        cases.append((bytes(b), 11, d, 0))
    check(emul, cases)


def test_names_of_every_length_at_every_phase(emul):
    cases = []
    for L in range(1, 301):
        name = bytes(0x61 + (i % 26) for i in range(L))
        for phase in range(0, 16, 3 if L > 40 else 1):
            s = b"\xab" * phase + cu.success(3, [name, b"z"]) + cu.success(4, [b"a", name])
            cases.append((s, 3, 2, phase))
    check(emul, cases)


def test_names_that_look_like_length_words(emul):
    names = [b"\x00\x00\x00\x05abcde", b"\x00\x00\x00\x01x", b"\x7f\xff\xff\xff", b"\x00\x00\x00\x10" + b"q" * 12,
             b"a\x00b", b"a/b", b".", b"..", b"...", b".a", b"\x00", b"/"]
    cases = []
    for k, n in enumerate(names):
        s = cu.success(9, [b"ok", n, b"tail"]) + cu.success(10, [n])
        cases.append((s, 9, 2, 0))
        cases.append((s[:len(s) - 1 - k % 3], 9, 2, 0))
    # a name whose bytes hold a complete entry: the chain skips it
    inner = struct.pack(">i", 3) + b"abc"
    cases.append((cu.success(9, [b"x" + inner, inner[::-1] + b"y"]) + cu.success(10, []), 9, 2, 0))
    check(emul, cases)


def test_counts(emul):
    cases = []
    for c in (-1, 0, 1, 2, 3, 100):
        body = struct.pack(">iqii", 5, 7, 0, c) + struct.pack(">i", 2) + b"ab" + struct.pack(">i", 1) + b"c"
        s = struct.pack(">i", len(body)) + body
        cases += [(s, 5, 1, 0), (cu.null_vector(5) + s, 5, 1, 0), (s + s, 5, 2, 0)]
    empty = struct.pack(">iqii", 5, 7, 0, 0)
    cases.append((struct.pack(">i", len(empty)) + empty, 5, 1, 0))
    big = struct.pack(">iqii", 5, 7, 0, 2 ** 31 - 1) + b"\0" * 40
    cases.append((struct.pack(">i", len(big)) + big, 5, 1, 0))
    check(emul, cases)
    assert want(*cases[-1])[1][0] == cu.SUCC_LEN
