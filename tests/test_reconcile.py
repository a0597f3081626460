"""Reconcile a batch with a snapshot of the registry (regk_reconcile) and frame the repairing requests
(regk_reconcile_requests).

CPU: the struct layout against the C compiler, and the clamped / two-buffer string helpers of regk_core.cuh against
Python, in a standalone g++ program built with AddressSanitizer so that a read past a buffer's end fails the test.
GPU: every output against the dictionary restatement in reconcile_util, on host and device snapshots, and the frames
against regk_jute_requests and pyoracle.
"""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import reconcile_util as ru

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZK_CREATE, ZK_DELETE, ZK_SETDATA = 1, 2, 5


# ------------------------------------------------------------------------------------------------------------ CPU --

def test_delta_struct_layout_matches_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(regk_delta), offsetof(regk_delta, m),
               offsetof(regk_delta, n_delete), offsetof(regk_delta, flags), offsetof(regk_delta, launches),
               offsetof(regk_delta, cls), offsetof(regk_delta, match), offsetof(regk_delta, obs_cls),
               offsetof(regk_delta, create), offsetof(regk_delta, dup), offsetof(regk_delta, del),
               offsetof(regk_delta, kernel_ms));
        printf("%d %d %d %d %d %d\n", REGK_DELTA_SAME, REGK_DELTA_CREATE, REGK_DELTA_UPDATE, REGK_DELTA_DUP,
               REGK_DELTA_KEEP, REGK_DELTA_DELETE);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    S = _native.CDelta
    assert got[:12] == [C.sizeof(S), S.m.offset, S.n_delete.offset, S.flags.offset, S.launches.offset, S.cls.offset,
                        S.match.offset, S.obs_cls.offset, S.create.offset, S.dup.offset, S.del_.offset, S.kernel_ms.offset]
    assert got[12:] == [ru.SAME, ru.CREATE, ru.UPDATE, ru.DUP, ru.KEEP, ru.DELETE]
    assert "regk_reconcile" in _native.EXPORTS and "regk_reconcile_requests" in _native.EXPORTS


def test_restatement_on_a_small_case():
    paths = [b"/a/x", b"/a/y", b"/a/x", b"/a/z", b"/a/w"]
    pays = [b"1", b"2", b"3", b"4", b""]
    nodes = [(b"/a/y", b"2"), (b"/a/x", b"9"), (b"/a/q", b""), (b"/a/w", b"")]
    r = ru.reconcile(paths, pays, nodes)
    assert r["cls"] == [ru.UPDATE, ru.SAME, ru.DUP, ru.CREATE, ru.SAME]
    assert r["match"] == [1, 0, 1, ru.NO_MATCH, 3] and r["obs_cls"] == [0, 0, 1, 0]
    assert (r["create"], r["update"], r["dup"], r["delete"]) == ([3], [0], [2], [2])
    with pytest.raises(ru.DuplicateNode) as e:
        ru.reconcile(paths, pays, nodes + [(b"/a/q", b"x")])
    assert e.value.index == 4


@pytest.fixture(scope="module")
def clamp_emul(built):
    """the helpers in a standalone program under AddressSanitizer (built in a temporary directory)"""
    d = tempfile.mkdtemp(prefix="regk_reconcile_emul")
    exe = os.path.join(d, "reconcile_emul")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-Wall", "-Wno-unknown-pragmas", "-fsanitize=address,undefined",
                           "-fno-sanitize-recover=all", "-fno-omit-frame-pointer", "-o", exe,
                           os.path.join(ROOT, "tests", "emul", "reconcile_emul.cpp")])

    def run(lines):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0", UBSAN_OPTIONS="halt_on_error=1")
        p = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, env=env)
        assert p.returncode == 0, p.stderr[-3000:]
        return [int(x) for x in p.stdout.split()]
    yield run
    import shutil
    shutil.rmtree(d, ignore_errors=True)


def _hex(b):
    return b.hex() if b else "-"


def test_clamped_helpers_match_python_at_every_phase(clamp_emul):
    rng = random.Random(21)
    lines, want = [], []
    for trial in range(600):
        n = rng.choice([0, 1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 33, 64, 100]) if trial % 4 else rng.randrange(0, 300)
        s = bytes(rng.randrange(256) for _ in range(n))
        pa, pb = rng.randrange(8), rng.randrange(8)
        tail_a = 0 if trial % 2 == 0 else rng.randrange(1, 6)        # half of them end exactly at the buffer's end
        tail_b = 0 if trial % 3 == 0 else rng.randrange(1, 6)
        A = bytes(rng.randrange(256) for _ in range(pa)) + s + bytes(rng.randrange(256) for _ in range(tail_a))
        kind = rng.randrange(4)
        t = s
        if kind == 1 and n:
            k = rng.choice([0, n - 1, rng.randrange(n)])              # one byte differs (the last one included)
            t = s[:k] + bytes([s[k] ^ (1 << rng.randrange(8))]) + s[k + 1:]
        B = bytes(rng.randrange(256) for _ in range(pb)) + t + bytes(rng.randrange(256) for _ in range(tail_b))
        lines += ["A " + _hex(A), "B " + _hex(B)]
        for k in range((n + 3) // 4 + 1):                             # every word of the string, and one past it
            lines.append("W %d %d" % (pa, k))
            want.append(int.from_bytes(A[pa + 4 * k:pa + 4 * k + 4].ljust(4, b"\0"), "little"))
        lines.append("H %d %d" % (pa, n))
        want.append(ru.string_hash32(s))
        lines.append("E %d %d %d" % (pa, pb, n))
        want.append(1 if s == t else 0)
    assert clamp_emul(lines) == want


def test_clamped_helpers_stop_at_the_buffer_end(clamp_emul):
    """strings that end exactly at a buffer's end at every length and phase: no read past it (AddressSanitizer), the
    same hash and equality as in a buffer with slack behind it"""
    lines, want = [], []
    for n in range(0, 21):
        for pa in range(0, 8):
            s = bytes((7 * i + n) & 0xFF for i in range(n))
            lines += ["A " + _hex(b"\x55" * pa + s), "B " + _hex(b"\xAA" * ((pa + 3) % 8) + s + b"\0" * 16)]
            lines.append("H %d %d" % (pa, n))
            want.append(ru.string_hash32(s))
            lines.append("E %d %d %d" % (pa, (pa + 3) % 8, n))
            want.append(1)
            lines.append("W %d %d" % (pa, n // 4))
            want.append(int.from_bytes(s[4 * (n // 4):].ljust(4, b"\0"), "little"))
    assert clamp_emul(lines) == want


# ------------------------------------------------------------------------------------------------------------ GPU --

@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def _dev(ctx, ptr, count, dtype):
    out = np.zeros(count, dtype)
    if count:
        assert ctx._lib.regk_memcpy_d2h(ctx._h, out.ctypes.data_as(C.c_void_p), C.c_void_p(ptr), out.nbytes) == 0
    return out


def _streams(res):
    return [res.path(i) for i in range(res.n)], [res.json(i) for i in range(res.n)]


def run(ctx, batch, **kw):
    """register `batch`; (paths, payloads) of its kept records"""
    got = ctx.register_batch(batch, **kw)
    paths, pays = _streams(got)
    if got.skipped is not None:
        drop = set(got.skipped.tolist())
        keep = [i for i in range(got.n) if i not in drop]
        paths, pays = [paths[i] for i in keep], [pays[i] for i in keep]
    return paths, pays


def device_snapshot(nodes):
    import torch
    from registrar_b200.batch import Snapshot
    h = Snapshot.from_nodes(nodes)
    t = lambda a, dt: torch.from_numpy(a.view(dt) if a.size else np.zeros(0, dt)).cuda()
    return Snapshot(t(h.path_bytes, np.uint8), t(h.path_off, np.int64), t(h.json_bytes, np.uint8), t(h.json_off, np.int64))


def check(ctx, paths, pays, nodes, frames=True, groups=(0,)):
    """ctx.reconcile over host and device snapshots of `nodes` against the restatement; the frames against pyoracle"""
    from registrar_b200.batch import Snapshot
    want = ru.reconcile(paths, pays, nodes)
    got = ctx.reconcile(Snapshot.from_nodes(nodes))
    assert got.n == len(paths) and got.m == len(nodes)
    assert got.cls.tolist() == want["cls"]
    assert got.match.tolist() == want["match"]
    assert got.obs_cls.tolist() == want["obs_cls"]
    for k in ("create", "update", "dup", "delete"):
        assert getattr(got, k).tolist() == want[k], k
    assert got.n_same == want["cls"].count(ru.SAME)
    raw = ctx.reconcile(device_snapshot(nodes), device=True)          # device snapshot, device outputs: the same
    assert np.array_equal(_dev(ctx, raw.cls, got.n, np.uint8), got.cls)
    assert np.array_equal(_dev(ctx, raw.match, got.n, np.uint64), got.match)
    assert np.array_equal(_dev(ctx, raw.obs_cls, got.m, np.uint8), got.obs_cls)
    for k, f in (("create", "create"), ("update", "update"), ("dup", "dup"), ("delete", "del_")):
        assert np.array_equal(_dev(ctx, getattr(raw, f), len(getattr(got, k)), np.uint64), getattr(got, k)), k
    if frames:
        sets = {ZK_CREATE: [(paths[i], pays[i]) for i in want["create"]],
                ZK_SETDATA: [(paths[i], pays[i]) for i in want["update"]],
                ZK_DELETE: [(nodes[j][0], b"") for j in want["delete"]]}
        for op, items in sets.items():
            for g in groups:
                fb, fo, _ = ctx.reconcile_requests(op, xid_base=7, group=g)
                assert fb.tobytes() == ru.frames(op, items, 7, g), (op, g)
                assert int(fo[-1]) == len(fb)
    return got


def drift(paths, pays, seed, frac=0.01):
    """a snapshot of the desired nodes with drift: nodes removed, payloads changed (one byte, the last byte, the
    length), empty data, foreign nodes (prefixes, extensions, last byte changed), shuffled"""
    rng = random.Random(seed)
    n = len(paths)
    k = max(1, int(n * frac))
    nodes = list(zip(paths, pays))
    idx = rng.sample(range(n), min(n, 8 * k))
    gone = set(idx[:k])
    for c, i in enumerate(idx[k:]):
        p, d = nodes[i]
        mode = c % 5
        if mode == 0 and d:
            j = rng.randrange(len(d))
            d = d[:j] + bytes([d[j] ^ 1]) + d[j + 1:]
        elif mode == 1 and d:
            d = d[:-1] + bytes([d[-1] ^ 0x20])
        elif mode == 2:
            d = d + b" " if c % 2 else d[:-1]
        elif mode == 3:
            d = b""
        else:
            continue
        nodes[i] = (p, d)
    nodes = [x for i, x in enumerate(nodes) if i not in gone]
    have = set(paths)
    for c, i in enumerate(rng.sample(range(n), min(n, k))):
        p = paths[i]
        for q in (p[:-1], p + b"x", p[:-1] + bytes([p[-1] ^ 1]), p + b"/child"):
            if q not in have:
                have.add(q)
                nodes.append((q, b"" if c % 3 == 0 else b"foreign"))
    rng.shuffle(nodes)
    return nodes


@pytest.mark.gpu
def test_identical_snapshot(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config1"))
    got = check(ctx, paths, pays, list(zip(paths, pays)), groups=(0, 7))
    assert got.n_same == got.n and got.n_create == got.n_update == got.n_dup == got.n_delete == 0
    for op in (ZK_CREATE, ZK_SETDATA, ZK_DELETE):
        fb, fo, _ = ctx.reconcile_requests(op)
        assert fb.size == 0 and fo.tolist() == [0]


@pytest.mark.gpu
@pytest.mark.parametrize("config,n", [("config1", None), ("config3", 1_000_000)])
def test_drift(ctx, config, n):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate(config, n=n))
    got = check(ctx, paths, pays, drift(paths, pays, seed=3), groups=(0, 100) if n else (0, 1, 7, 100))
    assert got.n_create > 0 and got.n_update > 0 and got.n_delete > 0 and got.n_dup == 0


def _var_host_records(n):
    return [{"domain": b"svc%d.dc%d.example.com" % (i % 41, i % 3), "hostname": b"h" * (1 + i % 37) + b"%d" % i,
             "type": b"host", "address": b"10.0.%d.%d" % (i % 200, i % 7)} for i in range(n)]


@pytest.mark.gpu
def test_drift_variable_hostnames_and_empty_snapshot(ctx):
    from registrar_b200.batch import RecordBatch
    batch = RecordBatch.from_records(_var_host_records(20_000))
    assert batch.host_off is not None
    paths, pays = run(ctx, batch)
    check(ctx, paths, pays, drift(paths, pays, seed=5, frac=0.05), groups=(0, 7))
    got = check(ctx, paths, pays, [], groups=(0, 100))                 # empty snapshot: every record is a create
    assert got.n_create == got.n
    fb, _, _ = ctx.reconcile_requests(ZK_CREATE, xid_base=2 ** 31 - 3, zk_flags=1)
    want, _, _ = ctx.jute_requests(ZK_CREATE, xid_base=2 ** 31 - 3, zk_flags=1)
    assert fb.tobytes() == want.tobytes()


@pytest.mark.gpu
def test_frames_equal_jute_requests_of_the_taken_records(ctx):
    from registrar_b200 import synth
    batch = synth.generate("config3", n=50_000, seed=17)
    paths, pays = run(ctx, batch)
    nodes = drift(paths, pays, seed=9, frac=0.03)
    d = check(ctx, paths, pays, nodes, frames=False)
    for g in (0, 1, 7, 100):
        for xid in (1, 2 ** 31 - 40):
            mine = {op: ctx.reconcile_requests(op, xid_base=xid, group=g, version=-1)[0].tobytes()
                    for op in (ZK_CREATE, ZK_SETDATA, ZK_DELETE)}
            ctx.register_batch(batch.take(d.create))                    # a later batch leaves the request streams alone
            assert mine[ZK_CREATE] == ctx.jute_requests(ZK_CREATE, xid_base=xid, group=g)[0].tobytes()
            ctx.register_batch(batch.take(d.update))
            assert mine[ZK_SETDATA] == ctx.jute_requests(ZK_SETDATA, xid_base=xid, group=g)[0].tobytes()
            assert mine[ZK_DELETE] == ru.frames(ZK_DELETE, [(nodes[j][0], b"") for j in d.delete], xid, g)
            assert mine[ZK_CREATE] == ctx.reconcile_requests(ZK_CREATE, xid_base=xid, group=g)[0].tobytes()


@pytest.mark.gpu
def test_duplicates_in_batch_and_snapshot(ctx):
    from registrar_b200 import _native
    from registrar_b200.batch import RecordBatch, Snapshot
    recs = [{"domain": b"svc%d.example.com" % (i % 5), "hostname": b"host%d" % (i % 200), "type": b"host",
             "address": b"10.1.1.%d" % i} for i in range(300)]
    paths, pays = run(ctx, RecordBatch.from_records(recs))
    nodes = [(p, d) for p, d in zip(paths[:60], pays[:60])][::2] + [(b"/com/example/gone", b"x")]
    got = check(ctx, paths, pays, nodes, groups=(0, 7))
    assert got.n_dup == 300 - 200 and got.dup.tolist() == list(range(200, 300))
    assert got.match[250] == got.match[50]
    bad = nodes + [nodes[3]]
    with pytest.raises(_native.RegkError) as e:
        ctx.reconcile(Snapshot.from_nodes(bad))
    assert e.value.code == 1 and "node %d " % (len(bad) - 1) in e.value.message
    with pytest.raises(_native.RegkError) as e:
        ctx.reconcile(device_snapshot(bad))
    assert e.value.code == 1 and "node %d " % (len(bad) - 1) in e.value.message
    with pytest.raises(_native.RegkError) as e:
        ctx.reconcile_requests(ZK_CREATE)                               # the failed call left no result
    assert e.value.code == 5


@pytest.mark.gpu
def test_alias_long_paths_and_tight_table(ctx):
    from registrar_b200 import synth
    from registrar_b200.batch import RecordBatch
    doms = [b"a.b", b"c.b", b"x." * 2500 + b"y", b"x." * 2500 + b"z", b"q.r.s", b"m." * 1100 + b"n"] * 3
    recs = [{"domain": d, "hostname": b"h", "type": b"host", "address": b"1.1.1.%d" % i} for i, d in enumerate(doms)]
    paths, pays = run(ctx, RecordBatch.from_records(recs, alias=True))
    assert max(len(p) for p in paths) > 4096
    nodes = [(paths[2], pays[2]), (paths[3], pays[3][:-1]), (paths[3][:-1], b""), (paths[2] + b"/k", b"")]
    got = check(ctx, paths, pays, nodes, groups=(0, 7))
    assert got.n_dup == len(doms) - 6
    ctx.set_option("reconcile_tight_table", 1)
    try:
        paths, pays = run(ctx, synth.generate("config3", n=100_000, seed=4))
        check(ctx, paths, pays, drift(paths, pays, seed=2, frac=0.02))
    finally:
        ctx.set_option("reconcile_tight_table", 0)


@pytest.mark.gpu
def test_dirty_skip_batch(ctx):
    from registrar_b200 import synth
    from registrar_b200.batch import RecordBatch
    base = synth.generate("config3", n=4000, seed=8)
    recs = [base.record(i) for i in range(base.n)]
    for i in (0, 5, 128, 1999, 3999):
        recs[i] = dict(recs[i], domain=recs[i]["domain"] + b"/x")
    paths, pays = run(ctx, RecordBatch.from_records(recs, types=base.types), skip_bad=True)
    assert len(paths) == base.n - 5
    check(ctx, paths, pays, drift(paths, pays, seed=4, frac=0.05))


@pytest.mark.gpu
def test_other_results_are_untouched(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=20_000, seed=12))
    raw = ctx.parent_dirs(device=True)
    n, nu = int(raw.n), int(raw.n_unique)
    before = (_dev(ctx, raw.parent_len, n, np.uint32), _dev(ctx, raw.unique_first, nu, np.uint64))
    dirs = ctx.mkdirp_dirs().dirs()
    frames = ctx.jute_requests(ZK_SETDATA, group=7)[0].tobytes()
    check(ctx, paths, pays, drift(paths, pays, seed=6))
    after = (_dev(ctx, raw.parent_len, n, np.uint32), _dev(ctx, raw.unique_first, nu, np.uint64))
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    assert ctx.mkdirp_dirs().dirs() == dirs
    assert ctx.jute_requests(ZK_SETDATA, group=7)[0].tobytes() == frames


@pytest.mark.gpu
def test_refusals(built):
    import torch
    from registrar_b200 import _native, synth
    from registrar_b200.batch import RecordBatch, Snapshot
    c = _native.Context(0)

    def refused(code, fn, text=None):
        with pytest.raises(_native.RegkError) as e:
            fn()
        assert e.value.code == code, e.value.message
        if text:
            assert text in e.value.message, e.value.message

    try:
        snap = Snapshot.from_nodes([(b"/a/b", b"x"), (b"/a/c", b"yy"), (b"/a/d", b"")])
        refused(5, lambda: c.reconcile(snap))                          # no batch yet
        refused(5, lambda: c.reconcile_requests())                     # no reconcile yet
        batch = synth.generate("config1")
        c.register_batch(batch, paths=False)
        refused(5, lambda: c.reconcile(snap))                          # REGK_NO_PATH
        c.register_batch(batch, payloads=False)
        refused(5, lambda: c.reconcile(snap))                          # REGK_NO_JSON
        c.register_batch(RecordBatch.from_records([], types=batch.types))
        refused(5, lambda: c.reconcile(snap))                          # an empty batch leaves no streams
        c.set_option("async", 1)
        t = c.submit(batch)
        refused(5, lambda: c.reconcile(snap))                          # a batch in flight
        c.collect(t)
        c.set_option("async", 0)
        d = c.reconcile(snap)
        assert d.n == batch.n and d.n_create == batch.n and d.n_delete == 3
        for op in (3, 0, 14):
            refused(1, lambda: c.reconcile_requests(op))
        cin, keep = snap.cdecode_in()
        for n in (2 ** 32 - 1, 2 ** 40):
            big = _native.CDecodeIn(n=n, flags=0, path_bytes=cin.path_bytes, path_off=cin.path_off,
                                    json_bytes=cin.json_bytes, json_off=cin.json_off)
            out = _native.CDelta()
            assert c._lib.regk_reconcile(c._h, C.byref(big), 0, C.byref(out)) == 1
        last = _native.CDecodeIn(n=3, flags=_native.FLAG_DECODE_LAST, path_bytes=cin.path_bytes, path_off=cin.path_off,
                                 json_bytes=cin.json_bytes, json_off=cin.json_off)
        assert c._lib.regk_reconcile(c._h, C.byref(last), 0, C.byref(_native.CDelta())) == 1
        # host offsets that are not monotone
        bad = Snapshot(snap.path_bytes, np.array([0, 4, 3, 12], np.uint64), snap.json_bytes, snap.json_off)
        refused(1, lambda: c.reconcile(bad), "node 1")
        # device snapshots: misaligned pointers, corrupt offsets (the smallest bad node is named, nothing is read)
        dev = device_snapshot([(b"/a/b%d" % i, b"v" * (i % 5)) for i in range(1000)])
        refused(1, lambda: c.reconcile(Snapshot(dev.path_bytes[1:], dev.path_off, dev.json_bytes, dev.json_off)), "misaligned")
        off8 = torch.zeros(dev.path_off.numel() + 1, dtype=torch.int64, device="cuda").view(torch.uint8)
        misaligned = off8[4:4 + 8 * dev.path_off.numel()]               # data_ptr 4 bytes into an allocation
        assert misaligned.data_ptr() % 8 == 4
        refused(1, lambda: c.reconcile(Snapshot(dev.path_bytes, misaligned, dev.json_bytes, dev.json_off)), "misaligned")
        ptot, jtot = dev.path_bytes.numel(), dev.json_bytes.numel()
        # (stream, entry, value): decreasing, past the total, huge, a reversed first node, past the payload total
        for which, j, v in (("path", 700, 3), ("path", 1000, ptot + 1), ("json", 400, 2 ** 62), ("path", 0, 2 ** 63 + 5),
                            ("json", 1000, jtot + 16)):
            po, jo = dev.path_off.clone(), dev.json_off.clone()
            (po if which == "path" else jo)[j] = v if v < 2 ** 63 else v - 2 ** 64
            with pytest.raises(_native.RegkError) as e:
                c.reconcile(Snapshot(dev.path_bytes, po, dev.json_bytes, jo))
            assert e.value.code == 1 and e.value.message.endswith("node %d" % max(j - 1, 0)), e.value.message
        po = dev.path_off.clone()
        po[300], po[200] = 10 ** 9, 1                                   # two bad places: the smaller is named
        with pytest.raises(_native.RegkError) as e:
            c.reconcile(Snapshot(dev.path_bytes, po, dev.json_bytes, dev.json_off))
        assert e.value.code == 1 and e.value.message.endswith("node 199"), e.value.message
        refused(5, lambda: c.reconcile_requests())                     # failed calls leave no result
        d = c.reconcile(dev)
        assert d.m == 1000 and d.n_delete == 1000
        assert len(c.reconcile_requests(ZK_DELETE)[1]) == 1001
    finally:
        c.set_option("async", 0)
        c.close()
