"""regk_read_results on the CPU: the restatement in results_util against replies worked out by hand from zookeeper.jute,
its server against the ZooKeeper model, and the per-frame and per-entry helpers of regk_results.cuh (results_head,
results_check, results_entry), compiled with g++ under AddressSanitizer, against the restatement's sequential reader:
every truncation point of a small stream, random streams with planted heads, well-formed streams with one byte changed,
and create paths whose bytes look like reply heads."""
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import reconcile_owned_util as ou
import reconcile_util as rcu
import results_util as su

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# CreateResponse to xid 5 for "/a", zxid 2^33 + 2^32, worked out by hand: len = 16 + 4 + 2 = 22
ONE_CREATE = bytes.fromhex("00000016" "00000005" "0000000300000000" "00000000" "00000002" "2f61")

# SetDataResponse to xid 6: Stat{czxid 2^32, mzxid 2^32 + 5, ctime 1.7e12 ms, mtime + 500, version 1, cversion 3,
# aversion 0, ephemeralOwner 0, dataLength 3, numChildren 0, pzxid 2^32 + 9}: len = 16 + 68 = 84
ONE_SETDATA = bytes.fromhex(
    "00000054" "00000006" "0000000300000000" "00000000"
    "0000000100000000" "0000000100000005" "0000018bcfe56800" "0000018bcfe569f4"
    "00000001" "00000003" "00000000" "0000000000000000" "00000003" "00000000" "0000000100000009")

# a three-operation multi (xid 7) rolled back by BADVERSION (-103) on its second operation: ErrorResults 0, -103, -2
# (MultiHeader{-1, false, e} ErrorResponse{e}, 13 bytes each), then MultiHeader{-1, true, -1}: len = 16 + 39 + 9 = 64
ONE_FAILED_MULTI = bytes.fromhex(
    "00000040" "00000007" "0000000300000000" "00000000"
    "ffffffff" "00" "00000000" "00000000"
    "ffffffff" "00" "ffffff99" "ffffff99"
    "ffffffff" "00" "fffffffe" "fffffffe"
    "ffffffff" "01" "ffffffff")


def offsets(fb):
    """the frame offsets of a request stream"""
    fo, pos = [0], 0
    while pos < len(fb):
        pos += 4 + int.from_bytes(fb[pos:pos + 4], "big")
        fo.append(pos)
    return fo


def test_builders_worked_out_by_hand():
    assert su._reply(5, 0, su.create_body(b"/a")) == ONE_CREATE
    n = ou.Node(b"xyz", 0)
    n.version = 1
    assert su._reply(6, 0, su.stat_of(n)) == ONE_SETDATA
    body = b"".join(su.mh(-1, False, c) + struct.pack(">i", c) for c in (0, su.BADVERSION, -2))
    assert su._reply(7, 0, body + su.mh(-1, True, -1)) == ONE_FAILED_MULTI
    assert su.error(9, su.NONODE) == bytes.fromhex("00000010" "00000009" "0000000300000000" "ffffff9b")
    fr = su.Framing(su.OP_SETDATA, [b"/p", b"/q", b"/r"], [3, 3, 3], xid_base=7, group=3)
    r = su.read(ONE_FAILED_MULTI, fr)
    assert r["cls"] == [su.ABORTED, su.FAILED, su.ABORTED] and r["err"] == [0, su.BADVERSION, -2]
    assert su.read(ONE_CREATE, su.Framing(su.OP_CREATE, [b"/a"], xid_base=5))["version"] == [0]
    assert su.read(ONE_SETDATA, su.Framing(su.OP_SETDATA, [b"/x"], [3], xid_base=6))["version"] == [1]


def test_server_answers_the_model():
    zk = ou.ZooKeeper()
    for p in (b"/a", b"/a/x", b"/a/y", b"/a/z"):
        zk.create(p, b"d", 0, ephemeral=False)
    srv = su.Server(zk, 77)
    # setData in groups of 2: the second frame's first entry has a stale version
    items = [(b"/a/x", b"new", 0), (b"/a/y", b"new", 0), (b"/a/z", b"new", 5), (b"/a", b"new", 0)]
    fb = ou.versioned_frames(su.OP_SETDATA, items, 3, group=2)
    s = srv.replies(fb, offsets(fb), extra={1: su.ping()})
    r = su.read(s, su.Framing(su.OP_SETDATA, [p for p, _, _ in items], [3] * 4, xid_base=3, group=2))
    assert r["cls"] == [su.DONE, su.DONE, su.FAILED, su.ABORTED] and r["err"] == [0, 0, su.BADVERSION, -2]
    assert r["version"] == [1, 1, -1, -1] and r["n_skipped"] == 1 and r["consumed"] == len(s)
    assert zk.nodes[b"/a/x"].data == b"new" and zk.nodes[b"/a/z"].data == b"d" and zk.nodes[b"/a"].version == 0
    # single deletes: NONODE counts as done, NOTEMPTY fails
    fb = rcu.frames(su.OP_DELETE, [(b"/a/x", b""), (b"/gone", b""), (b"/a", b"")], 10, 0)
    s = srv.replies(fb, offsets(fb))
    r = su.read(s, su.Framing(su.OP_DELETE, [b"/a/x", b"/gone", b"/a"], xid_base=10, tol=su.NONODE))
    assert r["cls"] == [su.DONE, su.DONE, su.FAILED] and r["err"] == [0, su.NONODE, su.NOTEMPTY]


@pytest.fixture(scope="module")
def emul(built):
    d = tempfile.mkdtemp(prefix="regk_results_emul")
    exe = os.path.join(d, "results_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "results_emul.cpp")])

    def run(cases):
        """cases = [(stream, Framing, start)] -> [(plausibility codes, read result)]"""
        lines = []
        for b, fr, start in cases:
            ents = " ".join("%s:%d" % (p.hex() or "-", d) for p, d in zip(fr.paths, fr.data_lens))
            lines += ["S %s" % (b.hex() or "-"),
                      "F %d %d %d %d %d %d %s" % (fr.xid_base, fr.op, fr.group, int(fr.multi), fr.tol, fr.entries, ents),
                      "P", "R %d" % start]
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        out = p.stdout.split("\n")
        return [([int(x) for x in out[2 * i].split()], out[2 * i + 1].split()) for i in range(len(cases))]
    yield run
    shutil.rmtree(d, ignore_errors=True)


def want(b, fr, start=0):
    codes = [su.plausible(b, pos, fr) for pos in range(len(b))]
    try:
        r = su.read(b, fr, start)
        ents = sum(([str(e), str(c), str(v)] for e, c, v in zip(r["err"], r["cls"], r["version"])), [])
        return codes, ["0", str(r["consumed"]), str(r["n_skipped"])] + [str(e) for e in r["frame_err"]] + ["|"] + ents
    except su.Refused as e:
        return codes, [str(e.code), str(e.pos), str(e.k)]


def check(emul, cases):
    for (s, fr, start), g in zip(cases, emul(cases)):
        assert g == want(s, fr, start), (s.hex(), fr.op, fr.group, start)


def scenario(op, group, xb=7, seed=1, clean=False):
    """a framing of `op` over eight nodes in groups of `group`, answered by the model: some writes fail, so some
    multi transactions roll back; clean=True: every write takes effect"""
    rng = random.Random(seed)
    zk = ou.ZooKeeper()
    zk.create(b"/d", b"", 0, ephemeral=False)
    paths = [b"/d/n%d" % i + b"x" * rng.randrange(0, 6) for i in range(8)]
    for i, p in enumerate(paths):
        if (i % 3 != 1 and not clean) or (clean and op != su.OP_CREATE):
            zk.create(p, b"old", 0, ephemeral=False)
    if op == su.OP_CREATE:
        fb = rcu.frames(op, [(p, b"pay%d" % i) for i, p in enumerate(paths)], xb, group, zk_flags=0)
        lens = [0] * 8
    elif op == su.OP_REPLACE:
        items = [(p, b"pay", 0 if i % 4 or clean else 3) for i, p in enumerate(paths)]
        fb = ou.replace_frames(items, xb, group, zk_flags=0)
        lens = [3] * 8
    else:
        items = [(p, b"data%d" % i, -1 if i % 5 or clean else 4) for i, p in enumerate(paths)]
        fb = ou.versioned_frames(op, items, xb, group)
        lens = [len(d) for _, d, _ in items]
    fo = offsets(fb)
    fr = su.Framing(op, paths, lens, xid_base=xb, group=group, tol=su.NONODE if op == su.OP_DELETE else 0)
    s = su.Server(zk, 5).replies(fb, fo, extra={0: su.ping(), 2: su.notification(b"/d")},
                                 header_err={1: -4} if fr.frames > 2 and not clean else None)
    return s, fr


SCENARIOS = [(op, g) for op in (su.OP_CREATE, su.OP_DELETE, su.OP_SETDATA) for g in (0, 1, 3)] + \
            [(su.OP_REPLACE, 1), (su.OP_REPLACE, 3)]


def test_scenarios_every_truncation_point(emul):
    cases = []
    for op, g in SCENARIOS:
        for clean in (False, True):
            s, fr = scenario(op, g, clean=clean)
            cases += [(s[:t], fr, 0) for t in range(len(s) + 1)]
            if clean:
                assert set(su.read(s, fr)["cls"]) == {su.DONE}
    check(emul, cases)
    outcomes = set()
    for op, g in SCENARIOS:
        s, fr = scenario(op, g)
        outcomes |= set(su.read(s, fr)["cls"])
    assert outcomes == {su.DONE, su.FAILED, su.ABORTED}


def test_random_streams_with_planted_heads(emul):
    rng = random.Random(5)
    cases = []
    for trial in range(300):
        op, g = rng.choice(SCENARIOS)
        _, fr = scenario(op, g, xb=rng.choice([0, 1, 2 ** 31 - 2, -2 ** 31, 1000]))
        ln = rng.randrange(0, 240)
        b = bytearray(rng.getrandbits(8) for _ in range(ln))
        if ln >= 40 and trial % 2:
            for _ in range(3):
                p = rng.randrange(0, ln - 39)
                k = rng.randrange(fr.frames)
                ok, bad = fr.lens(k)
                b[p:p + 4] = struct.pack(">i", rng.choice([16, ok, bad or ok, ln - p - 4, rng.randrange(-5, 200)]))
                b[p + 4:p + 8] = struct.pack(">i", rng.choice([su.wrap(fr.xid_base + k), -1, -2, -3]))
                b[p + 16:p + 20] = struct.pack(">i", rng.choice([0, 0, su.NONODE]))
                b[p + 20:p + 24] = struct.pack(">i", rng.choice([-1, 1, 2, 5]))
        cases.append((bytes(b), fr, min(rng.choice([0, 0, 1, 5]), ln)))
    # well-formed streams with one byte changed
    for _ in range(400):
        op, g = rng.choice(SCENARIOS)
        base, fr = scenario(op, g, seed=rng.randrange(4), clean=rng.random() < 0.5)
        b = bytearray(base)
        b[rng.randrange(len(b))] = rng.choice([0, 1, 0xFF, 0xFE, rng.getrandbits(8)])
        cases.append((bytes(b), fr, 0))
    check(emul, cases)


def test_create_paths_that_look_like_reply_heads(emul):
    """paths whose bytes hold a complete reply frame to another xid of the framing: the chain reads them as paths"""
    cases = []
    for g in (0, 2):
        head = su.error(8, su.NODEEXISTS)
        paths = [b"/" + head + b"%d" % i for i in range(4)]
        fb = rcu.frames(su.OP_CREATE, [(p, b"") for p in paths], 7, g, zk_flags=0)
        s = su.Server(ou.ZooKeeper(), 1).replies(fb, offsets(fb))
        fr = su.Framing(su.OP_CREATE, paths, xid_base=7, group=g)
        for phase in range(0, 16, 5):
            cases.append((b"\x00" * phase + s, fr, phase))
        cases.append((s[:-1], fr, 0))
        # a path echo that differs in its last byte
        bad = bytearray(s)
        bad[24 + (9 if g else 0) + len(paths[0]) - 1] ^= 1
        cases.append((bytes(bad), fr, 0))
    check(emul, cases)
    assert any(want(*c)[1][0] == str(su.PATH_ECHO) for c in cases)
