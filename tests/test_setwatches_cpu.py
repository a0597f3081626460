"""The SetWatches pieces without a GPU: the frames and the reply worked out by hand against the restatement in
setwatches_util, the model's DataTree.setWatches, the struct layouts against include/regk.h, and regk_setwatches.cuh's
host + device helpers - the reader's test with SetWatches replies (ev_sw_head / ev_sw_mask16) and the frame and entry
positions - compiled with g++ under AddressSanitizer against the restatement."""
import os
import random
import shutil
import struct
import subprocess
import tempfile

import pytest

import events_util as eu
import setwatches_util as sw
import stats_util as su

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_frame_and_reply_worked_out_by_hand():
    b, off = sw.frames([b"/a"], [b"/bb"], [], 0x10, 0, 3)
    assert b == bytes.fromhex("00000029" "fffffff8" "00000065" "0000000000000010" "00000001" "00000002" "2f61"
                              "00000001" "00000003" "2f6262" "00000000")
    assert off == [0, 45] and sw.parse(b) == [(0x10, [b"/a"], [b"/bb"], [])]
    assert sw.reply(0x100000005) == bytes.fromhex("00000010" "fffffff8" "0000000100000005" "00000000")
    # the split: B = 32 + 2 x (4 + 3) - 32 - 7 = 7, so each 6- or 7-byte entry opens a frame of its own
    assert [len(sum(f, [])) for f in sw.split([b"/a", b"/b"], [b"/cc"], [b"/d"], 32 + 14, 3)] == [2, 1, 1]


def test_setwatches_model_worked_out_by_hand():
    zk = sw.SessionZooKeeper()
    zk.create(b"/s", b"", 1, ephemeral=False)
    zk.create(b"/s/a", b"x", 1)
    zk.create(b"/s/b", b"y", 1)
    rel = zk.zxid
    zk.set_data(b"/s/a", b"z")
    zk.delete(b"/s/b")
    zk.drop_connection(1)
    s = zk.serve_setwatches(sw.frames([b"/s/a", b"/s/b"], [b"/s/c"], [b"/s", b"/t"], rel, 0, 4)[0], 1)
    r = sw.read(s, gate=True)
    assert r["n_events"] == 4 and r["n_replies"] == 1 and r["mark"] == zk.zxid
    got = [(t, p) for _, t, _, _, p in eu.read(s[:-20])["events"]]
    assert got == [(eu.DATA_CHANGED, b"/s/a"), (eu.DELETED, b"/s/b"), (eu.CHILDREN_CHANGED, b"/s"), (eu.DELETED, b"/t")]
    assert zk.data_w[1] == {b"/s/c"} and zk.child_w[1] == set()
    zk.create(b"/s/c", b"", 1)                                      # the re-armed exist watch fires
    assert [(t, p) for _, t, _, _, p in eu.read(zk.take_events(1))["events"]] == [(eu.CREATED, b"/s/c")]


def test_struct_layouts_match_header(built):
    import ctypes as C
    from registrar_b200 import _native
    d = tempfile.mkdtemp(prefix="regk_sw_abi")
    try:
        src = os.path.join(d, "t.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "regk.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu\\n",'
                    'sizeof(regk_setwatches_opts), sizeof(regk_setwatches), offsetof(regk_setwatches, n_dirty_dirs),'
                    'offsetof(regk_setwatches, relative_zxid), offsetof(regk_setwatches, frames), '
                    'offsetof(regk_setwatches, frames.kernel_ms));return 0;}\n')
        exe = os.path.join(d, "t")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", exe, src])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    finally:
        shutil.rmtree(d, ignore_errors=True)
    S = _native.CSetWatches
    assert got == [C.sizeof(_native.CSetWatchesOpts), C.sizeof(S), S.n_dirty_dirs.offset, S.relative_zxid.offset,
                   S.frames.offset, S.frames.offset + _native.CFrames.kernel_ms.offset]
    assert "regk_setwatches_requests" in _native.EXPORTS


@pytest.fixture(scope="module")
def emul():
    d = tempfile.mkdtemp(prefix="regk_sw_emul")
    exe = os.path.join(d, "setwatches_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "setwatches_emul.cpp")])

    def run(lines):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        return p.stdout.split("\n")
    yield run
    shutil.rmtree(d, ignore_errors=True)


def stream(seed, xb=7, n=4):
    rng = random.Random(seed)
    parts = []
    for _ in range(10):
        c = rng.randrange(6)
        if c == 0:
            parts.append(eu.ping())
        elif c == 1:
            parts.append(su.error(su.wrap(xb + rng.randrange(n)), su.NONODE))
        elif c == 2:
            parts.append(eu.notification(b"/s/n%d" % rng.randrange(100), 3))
        elif c == 3:
            parts.append(sw.reply(rng.getrandbits(40)))
        elif c == 4:
            parts.append(sw.reply(5, err=rng.choice([0, -4]), body=rng.choice([b"", b"\0" * 4])))
        else:
            parts.append(sw.reply(9)[:rng.randrange(1, 20)])
    return b"".join(parts)


def test_head_and_mask_against_the_restatement(emul):
    cases = [stream(k) for k in range(30)] + [sw.reply(3), sw.reply(3, err=1), sw.reply(3, body=b"x"), b""]
    lines = []
    for b in cases:
        lines += ["S %s" % (b.hex() or "-"), "X 7 4", "P", "M"]
    out = emul(lines)
    for i, b in enumerate(cases):
        codes = [sw.head(b, pos, 7, 4, True) for pos in range(len(b))]
        assert [int(x) for x in out[2 * i].split()] == codes, b.hex()
        assert [int(x) for x in out[2 * i + 1].split()] == [int(c == eu.OK) for c in codes], b.hex()


def test_entry_and_frame_positions_against_the_restatement(emul):
    rng = random.Random(4)
    lines, want = [], []
    for _ in range(40):
        lmax = rng.randrange(1, 40)
        mf = 32 + 2 * (4 + lmax) + rng.choice([0, 1, 5, 200])
        lists = [[b"/" + b"p" * rng.randrange(0, lmax) for _ in range(rng.randrange(0, 12))] for _ in range(3)]
        b, off = sw.frames(*lists, 5, mf, lmax)
        B = mf - 32 - 4 - lmax
        at = []                                                     # every entry's position, walking the frames
        for f in range(len(off) - 1):
            k = off[f] + 20
            for _ in range(3):
                (cnt,) = struct.unpack_from(">i", b, k)
                k += 4
                for _ in range(cnt):
                    at.append(k)
                    k += 4 + struct.unpack_from(">i", b, k)[0]
        s, firsts, j = 0, [], 0
        for lst, paths in enumerate(lists):
            pos, exp = [], []
            for p in paths:
                pos.append(s)
                exp.append(at[j])
                j += 1
                if not firsts or s // B != firsts[-1][0]:
                    firsts.append((s // B, s))
                s += 4 + len(p)
            if pos:
                lines.append("E %d %d %s" % (B, lst, " ".join(map(str, pos))))
                want.append(exp)
        for f, s0 in firsts:
            lines.append("F %d %d" % (f, s0))
            want.append([off[f]])
    out = emul(lines)
    for k, exp in enumerate(want):
        assert [int(x) for x in out[k].split()] == exp, k
