"""The watched heartbeat on the CPU: the restatement in events_util against a notification and watch-byte frames worked
out by hand, and the watch-aware ZooKeeper model against a create, a delete and a replace multi; the struct layouts
against the C compiler; and the helpers of regk_events.cuh (ev_head, and ev_mask16, the candidate test from registers),
compiled with g++ under AddressSanitizer, against the restatement: every position's verdict and a front-to-back walk
over every truncation point, path lengths at every 16-byte phase, random streams with planted heads, paths that look
like length words, and reply frames in range mixed in."""
import ctypes as C
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import events_util as eu
import reconcile_owned_util as ou
import stats_util as su

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S1 = 0x1234_5678_9ABC_DEF0

# WatcherEvent{NodeDataChanged, SyncConnected, "/a/b"} with zxid 2^32 + 7: len = 16 + 12 + 4
ONE_EVENT = bytes.fromhex("00000020" "ffffffff" "0000000100000007" "00000000" "00000003" "00000003" "00000004" "2f612f62")
# ExistsRequest{"/a", watch = true} with xid 5, GetChildrenRequest{"/a", watch = true} with xid 6
ONE_EXISTS = bytes.fromhex("0000000f" "00000005" "00000003" "00000002" "2f61" "01")
ONE_CHILDREN = bytes.fromhex("0000000f" "00000006" "00000008" "00000002" "2f61" "01")


def test_frames_worked_out_by_hand():
    assert eu.notification(b"/a/b", eu.DATA_CHANGED, zxid=2 ** 32 + 7) == ONE_EVENT
    assert eu.read_frames(3, [b"/a"], 5, watch=True) == ONE_EXISTS
    assert eu.read_frames(8, [b"/a"], 6, watch=True) == ONE_CHILDREN
    assert eu.read_frames(3, [b"/a"], 5) == su.exists_frames([b"/a"], 5)             # watch = false: the frames of today
    r = eu.read(eu.ping() + su.error(9, su.NONODE) + ONE_EVENT + ONE_EVENT[:7], 9, 1)
    assert r["events"] == [(40, 3, 3, 2 ** 32 + 7, b"/a/b")] and r["n_pings"] == 1 and r["n_replies"] == 1
    assert r["consumed"] == 76 and r["partial"]
    with pytest.raises(eu.Refused) as e:
        eu.read(su.error(9, su.NONODE), 10, 1)
    assert (e.value.code, e.value.pos) == (eu.XID_RANGE, 0)
    m = eu.Mapper([b"/s/a", b"/s/b", b"/s/a", b"/t/c"])
    got, unmatched, other = m.feed([(0, eu.DATA_CHANGED, 3, 0, b"/s/a"), (0, eu.CHILDREN_CHANGED, 3, 0, b"/t"),
                                    (0, eu.DELETED, 3, 0, b"/s"), (0, 5, 3, 0, b"/s/b"), (0, eu.CREATED, 3, 0, b"/x")])
    assert got == [(1, 0), (2, 1), (2, 0), (0, eu.NO_SUBJECT), (0, eu.NO_SUBJECT)] and (unmatched, other) == (2, 1)
    assert m.take() == [0] and m.take(dirs=True) == [0, 1] and m.take() == []


def test_watch_model_worked_out_by_hand():
    zk = eu.WatchedZooKeeper()
    assert zk.create(b"/s", b"", 0, ephemeral=False) == ou.ZOK
    assert zk.create(b"/s/a", b"abc", S1) == ou.ZOK
    # arm: an exists on /s/a and on the missing /s/b, a getChildren on /s
    zk.serve_reads(eu.read_frames(3, [b"/s/a", b"/s/b"], 1, watch=True) + eu.read_frames(8, [b"/s"], 3, watch=True), S1)
    assert zk.take_events(S1) == b""
    # a create: NodeCreated on the node, NodeChildrenChanged on its parent; both watches are spent
    assert zk.create(b"/s/b", b"x", S1) == ou.ZOK
    r = eu.read(zk.take_events(S1))
    assert [(t, p) for _, t, _, _, p in r["events"]] == [(eu.CREATED, b"/s/b"), (eu.CHILDREN_CHANGED, b"/s")]
    assert zk.create(b"/s/c", b"x", S1) == ou.ZOK and zk.take_events(S1) == b""     # one-shot
    # a delete: NodeDeleted on the node; the parent's child watch is not armed any more
    assert zk.delete(b"/s/a") == ou.ZOK
    assert [(t, p) for _, t, _, _, p in eu.read(zk.take_events(S1))["events"]] == [(eu.DELETED, b"/s/a")]
    # a replace multi (delete + create of one node) fires per operation: its delete spends the node's watch and its
    # parent's, so its create finds none armed
    zk.serve_reads(eu.read_frames(3, [b"/s/b"], 9, watch=True) + eu.read_frames(8, [b"/s"], 10, watch=True), S1)
    fb = ou.replace_frames([(b"/s/b", b"yy", 0)], xid_base=20, group=1)
    assert zk.apply_frame(fb, S1) == ou.ZOK
    got = [(t, p) for _, t, _, _, p in eu.read(zk.take_events(S1))["events"]]
    assert got == [(eu.DELETED, b"/s/b"), (eu.CHILDREN_CHANGED, b"/s")]
    # a multi that fails fires nothing
    zk.serve_reads(eu.read_frames(3, [b"/s/b"], 30, watch=True), S1)
    bad = ou.replace_frames([(b"/s/b", b"z", 7)], xid_base=31, group=1)              # wrong version: rolled back
    assert zk.apply_frame(bad, S1) == ou.BADVERSION and zk.take_events(S1) == b""
    assert zk.set_data(b"/s/b", b"zzz") == ou.ZOK
    assert [(t, p) for _, t, _, _, p in eu.read(zk.take_events(S1))["events"]] == [(eu.DATA_CHANGED, b"/s/b")]
    # a watch without its byte is not armed; a directory deleted fires NodeDeleted through its child watch
    zk.serve_reads(eu.read_frames(3, [b"/s/c"], 40), S1)
    assert zk.set_data(b"/s/c", b"q") == ou.ZOK and zk.take_events(S1) == b""
    assert zk.create(b"/u", b"", 0, ephemeral=False) == ou.ZOK
    zk.serve_reads(eu.read_frames(8, [b"/u"], 41, watch=True), S1)
    assert zk.delete(b"/u") == ou.ZOK
    assert [(t, p) for _, t, _, _, p in eu.read(zk.take_events(S1))["events"]] == [(eu.DELETED, b"/u")]


def test_struct_layouts_match_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu ", sizeof(regk_events_opts), offsetof(regk_events_opts, n_xids),
               offsetof(regk_events_opts, flags), sizeof(regk_events), offsetof(regk_events, consumed));
        printf("%zu %zu %zu %zu %zu %zu %zu %zu %u %u %u\n", offsetof(regk_events, n_dirty_dirs),
               offsetof(regk_events, partial), offsetof(regk_events, launches), offsetof(regk_events, pos),
               offsetof(regk_events, subject_kind), offsetof(regk_events, subject), offsetof(regk_events, kernel_ms),
               offsetof(regk_events, type), REGK_ZK_WATCH, REGK_EV_RECORD, REGK_EV_DIR);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    O, E = _native.CEventsOpts, _native.CEvents
    assert got == [C.sizeof(O), O.n_xids.offset, O.flags.offset, C.sizeof(E), E.consumed.offset, E.n_dirty_dirs.offset,
                   E.partial.offset, E.launches.offset, E.pos.offset, E.subject_kind.offset, E.subject.offset,
                   E.kernel_ms.offset, E.type.offset, _native.FLAG_ZK_WATCH, _native.EV_RECORD, _native.EV_DIR]
    assert "regk_read_events" in _native.EXPORTS and "regk_events_requests" in _native.EXPORTS


@pytest.fixture(scope="module")
def emul(built):
    d = tempfile.mkdtemp(prefix="regk_events_emul")
    exe = os.path.join(d, "events_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "events_emul.cpp")])

    def run(cases):
        """cases = [(stream, xid_base, n, start)] -> [(head codes, mask bits, walk result)]"""
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
    codes = [eu.head(b, pos, xb, n) for pos in range(len(b))]
    mask = [int(c == eu.OK and pos >= start) for pos, c in enumerate(codes)]
    try:
        r = eu.read(b, xb, n, start)
        evs = sum(([str(pos), str(t), str(st), str(z), str(len(p))] for pos, t, st, z, p in r["events"]), [])
        return codes, mask, ["0", str(r["consumed"]), str(int(r["partial"])), str(r["n_pings"]), str(r["n_replies"])] + evs
    except eu.Refused as e:
        return codes, mask, [str(e.code), str(e.pos)]


def check(emul, cases):
    for c, g in zip(cases, emul(cases)):
        assert g == want(*c), (c[0].hex(), c[1:])


def scenario(xb=7, seed=1, n=6):
    """notifications of every type, pings and in-range replies interleaved"""
    rng = random.Random(seed)
    parts = []
    for k in range(12):
        c = rng.randrange(4)
        if c == 0:
            parts.append(eu.ping())
        elif c == 1:
            parts.append(su.error(su.wrap(xb + rng.randrange(n)), su.NONODE) if rng.randrange(2) else
                         su.success(su.wrap(xb + rng.randrange(n)), 1, 2, 3, seed=k))
        else:
            parts.append(eu.notification(b"/s/n%d" % rng.randrange(100), rng.randrange(-1, 8), zxid=rng.getrandbits(40)))
    return b"".join(parts)


def test_every_truncation_point_and_start_phase(emul):
    s = scenario()
    r = eu.read(s, 7, 6)
    assert r["events"] and r["n_pings"] and r["n_replies"] and not r["partial"]
    cases = [(s[:t], 7, 6, 0) for t in range(len(s) + 1)]
    for phase in range(17):
        cases.append((bytes(range(1, phase + 1)) + s, 7, 6, phase))
    for xb in (2 ** 31 - 4, -2 ** 31, 0):
        cases.append((scenario(xb), xb, 6, 0))
    check(emul, cases)


def test_path_lengths_at_every_phase(emul):
    cases = []
    for plen in range(0, 40):
        for lead in range(16):
            path = bytes(b"/abcdefghijklmnopqrstuvwxyz0123456789ABCDEFGH"[:plen])
            s = eu.ping()[:0] + b"\x00" * 0 + eu.notification(path, eu.CHILDREN_CHANGED)
            cases.append((bytes([0xAB]) * lead + s + eu.ping(), 0, 0, lead))
    check(emul, cases)


def test_random_streams_with_planted_heads(emul):
    rng = random.Random(5)
    cases = []
    for trial in range(400):
        xb = rng.choice([0, 1, 2 ** 31 - 2, -2 ** 31, 1000])
        n = rng.choice([0, 1, 3, 8, 2 ** 31])
        ln = rng.randrange(0, 260)
        b = bytearray(rng.getrandbits(8) for _ in range(ln))
        if ln >= 36 and trial % 2:
            for _ in range(4):
                p = rng.randrange(0, ln - 35)
                L = rng.choice([16, 28, 31, ln - p - 4, 15, rng.randrange(-5, 200)])
                b[p:p + 4] = struct.pack(">i", L)
                b[p + 4:p + 8] = struct.pack(">i", rng.choice([su.wrap(xb + rng.randrange(max(1, min(n, 9)))), -1, -1, -2, -3]))
                b[p + 16:p + 20] = struct.pack(">i", rng.choice([0, 0, 0, 1]))
                b[p + 20:p + 24] = struct.pack(">i", rng.choice([-1, 1, 4, 7, 8, -2]))
                b[p + 28:p + 32] = struct.pack(">i", rng.choice([L - 28, L - 28, -1, L - 27]))
        cases.append((bytes(b), xb, n, min(rng.choice([0, 0, 1, 5, 16, 17]), ln)))
    for _ in range(300):
        b = bytearray(scenario(seed=rng.randrange(4)))
        b[rng.randrange(len(b))] = rng.choice([0, 1, 0xFF, 0xFE, 0x80, rng.getrandbits(8)])
        cases.append((bytes(b), 7, 6, 0))
    # each refusal on its own
    cases += [(eu.notification(b"/a", err=-4), 0, 0, 0), (eu.notification(b"/a", typ=8), 0, 0, 0),
              (eu.notification(b"/a", typ=-2), 0, 0, 0), (eu.notification(b"/abc", plen=-1), 0, 0, 0),
              (eu.notification(b"/abc", plen=2), 0, 0, 0), (su.error(-2, 0) + b"\0" * 4, 0, 0, 0),
              (su.error(-3, 0), 0, 0, 0), (su.error(5, 0), 0, 5, 0), (b"\0\0\0\x0f" + b"\0" * 15, 0, 0, 0)]
    bad = bytearray(su.error(-2, 0))
    bad[0:4] = struct.pack(">i", 20)
    cases.append((bytes(bad) + b"\0" * 4, 0, 0, 0))
    check(emul, cases)
    assert {want(*c)[2][0] for c in cases} >= {str(k) for k in (eu.OK, eu.BAD_LEN, eu.NEG_XID, eu.XID_RANGE, eu.NOTE_LEN,
                                                               eu.NEG_PATH, eu.NOTE_ERR, eu.TYPE, eu.PING_BODY)}


def test_paths_that_look_like_length_words_and_replies(emul):
    """notification paths that hold whole frames - pings, notifications, in-range replies: every position inside is
    plausible on its own, and the walk steps over the whole notification"""
    inner = eu.ping() + eu.notification(b"/q", 2) + su.error(8, su.NONODE) + su.success(9, 3, 0, 5, seed=9)
    cases = []
    for phase in (0, 1, 7, 15):
        s = eu.notification(b"/" + inner, eu.DATA_CHANGED) + su.error(7, su.NONODE) + eu.notification(b"/" + inner * 3, 1)
        cases.append((b"\x00" * phase + s, 7, 3, phase))
    check(emul, cases)
    codes = want(*cases[0])[0]
    assert sum(c == eu.OK for c in codes) > 6
