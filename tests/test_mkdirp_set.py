"""The mkdirp set of a batch (regk_mkdirp_dirs) and its CreateRequest frames (regk_mkdirp_requests).

CPU: the restatement in mkdirp_util agrees with the executed reference's mkdirp calls, and the host+device helpers of
regk_core.cuh (compiled with g++ through tests/emul/mkdirp_emul.cpp) agree with the restatement.
GPU: the set, its order, depth_off, the packed bytes and the invalid list equal the restatement on every kind of
batch, and the frames equal pyoracle's CreateRequest of each directory.
"""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

from mkdirp_util import ancestors, components, dir_of, mkdirp_frames, mkdirp_set
from oracle import pyoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------ CPU --

def _node_paths(d):
    """the nodes register() writes for one fixture input: the host node, then one alias node per alias"""
    paths = [pyoracle.host_node_path(d["domain"], d["hostname"])]
    paths += [pyoracle.domain_to_path(a) for a in d.get("aliases") or []]
    return [p.encode("latin-1") for p in paths]


def test_restatement_follows_the_reference_mkdirp_calls():
    from golden_util import load
    seen_invalid = 0
    for row in load("calls.jsonl"):
        paths = _node_paths(row["in"])
        args = [c[1].encode("latin-1") for c in row["calls"] if c[0] == "mkdirp"]
        assert args == [dir_of(p) for p in paths]           # one mkdirp per node, of path.dirname (pins dir_of)
        dirs, first, invalid = mkdirp_set(paths)
        want = set()
        for a in args:
            if components(a) is None:
                continue
            want.update(ancestors(a))
        assert set(dirs) == want and len(dirs) == len(want)   # every valid argument and every ancestor, nothing else
        assert sorted({dir_of(paths[i]) for i in invalid}) == sorted({a for a in args if components(a) is None})
        seen_invalid += len(invalid)
        for k, d in enumerate(dirs):                          # parents first
            assert all(dirs.index(a) < k for a in ancestors(d)[:-1])
            assert paths[first[k]].startswith(d)
    assert seen_invalid == 1                                  # '/b/' of the alias a..b


@pytest.fixture(scope="module")
def mkemul(built):
    so = os.path.join(ROOT, "tests", "emul", "libmkdirpemul.so")
    srcs = [os.path.join(ROOT, "tests", "emul", "mkdirp_emul.cpp"), os.path.join(ROOT, "registrar_b200", "csrc", "regk_core.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(f) for f in srcs):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                               "-fsanitize=undefined", "-fno-sanitize-recover=undefined", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emul_mkdirp.restype = C.c_uint64
    return lib


def _emul(lib, dirs):
    off = np.zeros(len(dirs) + 1, np.uint64)
    np.cumsum([len(d) for d in dirs], out=off[1:])
    raw = np.frombuffer(b"".join(dirs) + b"\0" * 8, np.uint8).copy()
    comps = np.zeros(len(dirs), np.uint32)
    cap = sum(len(d) for d in dirs) + 1
    ends, hashes = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    w = lib.emul_mkdirp(p(raw), p(off), len(dirs), p(comps), p(ends), p(hashes))
    return comps, ends[:w], hashes[:w]


def _check_helpers(lib, dirs):
    comps, ends, hashes = _emul(lib, dirs)
    w, by_prefix = 0, {}
    for k, d in enumerate(dirs):
        c = components(d)
        assert int(comps[k]) == (0xFFFFFFFF if c is None else c), d
        want = [len(a) for a in ancestors(d)]
        assert ends[w:w + len(want)].tolist() == want, d
        for a, h in zip(ancestors(d), hashes[w:w + len(want)]):
            assert by_prefix.setdefault(a, int(h)) == int(h)     # the hash of a prefix depends on its bytes alone
        w += len(want)
    assert w == len(ends)
    return comps


EDGE_DIRS = [b"", b"/", b"//", b"///", b"/a", b"/a/", b"/a//b", b"//a", b"/a/b/c", b"/b/", b"/\x00", b"/a\x1f/b", b"/a\x7f",
             b"/a\x20b", b"/~/!", b"a/b", b"/" + b"x" * 300, b"/" + b"/".join(b"c%d" % i for i in range(100)), b"/a/b/"]


def test_helpers_match_the_restatement_on_the_edge_fixtures(mkemul):
    from golden_util import as_record, load
    recs = [as_record(r["in"]) for r in load("edge.jsonl")]
    dirs = list(EDGE_DIRS)
    for r in recs:
        dom = r["domain"].decode("latin-1")
        dirs.append(dir_of(pyoracle.domain_to_path(dom).encode("latin-1")))
        try:
            dirs.append(dir_of(pyoracle.host_node_path(dom, r["hostname"].decode("latin-1")).encode("latin-1")))
        except Exception:
            pass
    comps = _check_helpers(mkemul, dirs)
    assert (comps == 0xFFFFFFFF).sum() >= 8 and (comps > 64).any()


def _random_dir(rng):
    kind = rng.random()
    n = rng.choice([1, 2, 3, 5, 8, 65, 70, 130]) if kind < 0.9 else rng.randrange(0, 4)
    comps = []
    for _ in range(n):
        c = bytes(rng.choice(b"abcxyz-_09.") for _ in range(rng.randrange(1, 6)))
        r = rng.random()
        if r < 0.04:
            c = b""                                             # empty component
        elif r < 0.08:
            c = c + bytes([rng.choice([0x00, 0x01, 0x1F, 0x7F, 0x09])])     # control byte
        comps.append(c)
    d = b"/" + b"/".join(comps)
    r = rng.random()
    if r < 0.05:
        d += b"/"                                               # trailing '/'
    elif r < 0.1:
        d = b"/" + d                                            # '//x' root
    elif r < 0.12:
        d = d[1:]                                               # no leading '/'
    return d


def test_helpers_match_the_restatement_on_random_paths(mkemul):
    rng = random.Random(5)
    dirs = [_random_dir(rng) for _ in range(4000)]
    dirs += [d[:k] for d in dirs[:200] for k in (len(d) // 2, len(d) - 1)]      # prefixes of the same strings
    comps = _check_helpers(mkemul, dirs)
    assert (comps == 0xFFFFFFFF).sum() > 400 and (comps > 64).sum() > 100 and (comps == 0).sum() > 0


def test_dirs_struct_layout_matches_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(regk_dirs), offsetof(regk_dirs, max_depth),
               offsetof(regk_dirs, dir_rec), offsetof(regk_dirs, depth_off), offsetof(regk_dirs, invalid),
               offsetof(regk_dirs, dir_bytes_len), offsetof(regk_dirs, kernel_ms), offsetof(regk_dirs, closure_ms),
               offsetof(regk_dirs, gather_ms));
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    S = _native.CDirs
    assert got == [C.sizeof(S), S.max_depth.offset, S.dir_rec.offset, S.depth_off.offset, S.invalid.offset,
                   S.dir_bytes_len.offset, S.kernel_ms.offset, S.closure_ms.offset, S.gather_ms.offset]
    assert "regk_mkdirp_dirs" in _native.EXPORTS and "regk_mkdirp_requests" in _native.EXPORTS


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


def _device_set(ctx):
    raw = ctx.mkdirp_dirs(device=True)
    nd, ni, md = int(raw.n_dirs), int(raw.n_invalid), int(raw.max_depth)
    return (_dev(ctx, raw.dir_rec, nd, np.uint64), _dev(ctx, raw.dir_len, nd, np.uint32),
            _dev(ctx, raw.depth_off, md + 1, np.uint64), _dev(ctx, raw.dir_bytes, int(raw.dir_bytes_len), np.uint8),
            _dev(ctx, raw.dir_off, nd + 1, np.uint64), _dev(ctx, raw.invalid, ni, np.uint64))


def check_set(ctx, paths, frames=True):
    """the set of the batch finished last on ctx against the restatement over its (kept) node paths"""
    dirs, first, invalid = mkdirp_set(paths)
    ds = ctx.mkdirp_dirs()
    assert ds.n == len(paths)
    assert ds.dirs() == dirs
    assert ds.dir_rec.tolist() == first
    assert ds.dir_len.tolist() == [len(d) for d in dirs]
    depth = [d.count(b"/") for d in dirs]
    want_off = [0] + [sum(1 for x in depth if x <= k) for k in range(1, (max(depth) if depth else 0) + 1)]
    assert ds.depth_off.tolist() == want_off and ds.max_depth == len(want_off) - 1
    assert ds.dir_off[-1] == len(ds.dir_bytes)
    assert ds.invalid.tolist() == invalid
    again = ctx.mkdirp_dirs()                                   # no atomics leak into the order
    assert again.dirs() == dirs and np.array_equal(again.dir_rec, ds.dir_rec) and np.array_equal(again.dir_off, ds.dir_off)
    dev = _device_set(ctx)
    for a, b in zip(dev, (ds.dir_rec, ds.dir_len, ds.depth_off, ds.dir_bytes, ds.dir_off, ds.invalid)):
        assert np.array_equal(a, b)
    if frames:
        fb, fo, _ = ctx.mkdirp_requests()
        assert fb.tobytes() == mkdirp_frames(dirs, 1, 0)
        assert len(fo) == len(dirs) + 1 and int(fo[-1]) == len(fb)
    return ds


def _paths(res):
    return [res.path(i) for i in range(res.n)]


def _run(ctx, batch, **kw):
    from oracle import oracle
    got = ctx.register_batch(batch, **kw)
    want = oracle.register_batch(batch)
    paths = _paths(want)
    assert _paths(got) == paths
    return paths


@pytest.mark.gpu
@pytest.mark.parametrize("config,n", [("config1", None), ("config2", None), ("config3", 300_000)])
def test_synthetic_host_batches(ctx, config, n):
    from registrar_b200 import synth
    check_set(ctx, _run(ctx, synth.generate(config, n=n)), frames=config != "config2")


def fleet(n, ndom=1000, seed=3):
    """n config 2 records collapsed onto the domains of the first `ndom` (tools/parents_time.py's fleet case)"""
    from registrar_b200 import synth
    rng = np.random.default_rng(seed)
    b = synth.generate("config2", n=n)
    idx = rng.integers(0, ndom, n)
    lens = np.diff(b.domain_off)[idx]
    off = np.zeros(n + 1, np.uint32)
    np.cumsum(lens, out=off[1:])
    src0 = b.domain_off[:-1][idx]
    pos = np.repeat(src0.astype(np.int64) - off[:-1].astype(np.int64), lens) + np.arange(int(off[-1]), dtype=np.int64)
    b.domain_bytes = b.domain_bytes[pos]
    b.domain_off = off
    return b


@pytest.mark.gpu
def test_fleet_batch(ctx):
    ds = check_set(ctx, _run(ctx, fleet(200_000)))
    assert 0 < ds.n_dirs < 4000


def _alias_records(doms):
    return [{"domain": d, "hostname": b"h", "type": b"host", "address": b"1.1.1.1"} for d in doms]


@pytest.mark.gpu
def test_alias_batches_with_empty_and_control_labels(ctx):
    from registrar_b200.batch import RecordBatch
    doms = [b"a.b", b"a..b", b"a.", b".a", b"", b"a", b"..", b"a.b.", b".a.b", b"x.y.z", b"x\x01.y.z", b"q.x\x7f.z",
            b"a...", b"..a..b..", b"c.b", b"x.y.z", b"w\x1f", b"b.a.b", b"m." * 70 + b"n"]
    rng = random.Random(11)
    doms += [b".".join(rng.choice([b"a", b"b", b"", b"c\x02", b"d"]) for _ in range(rng.randrange(1, 8))) for _ in range(3000)]
    batch = RecordBatch.from_records(_alias_records(doms), alias=True)
    ds = check_set(ctx, _run(ctx, batch))
    assert ds.invalid.size > 10 and ds.max_depth > 64
    host = RecordBatch.from_records([dict(r, hostname=b"h%d" % i) for i, r in enumerate(_alias_records(doms))])
    ds = check_set(ctx, _run(ctx, host))                        # host nodes: only control bytes make a directory invalid
    assert ds.invalid.size > 0


@pytest.mark.gpu
def test_variable_length_hostnames_and_tiny_batches(ctx):
    from registrar_b200.batch import RecordBatch
    recs = [{"domain": b"svc%d.dc%d.example.com" % (i % 41, i % 3), "hostname": b"h" * (1 + i % 37), "type": b"host",
             "address": b"10.0.0.1"} for i in range(5000)]
    batch = RecordBatch.from_records(recs)
    assert batch.host_off is not None
    check_set(ctx, _run(ctx, batch))
    check_set(ctx, _run(ctx, RecordBatch.from_records(recs[:1])))
    check_set(ctx, _run(ctx, RecordBatch.from_records(_alias_records([b""]), alias=True)))     # '/' only: empty set
    from registrar_b200._native import RegkError
    _run(ctx, RecordBatch.from_records(recs[:0], types=batch.types))
    with pytest.raises(RegkError) as e:
        ctx.mkdirp_dirs()                                       # an empty batch leaves no path stream, as for parent_dirs
    assert e.value.code == 5


@pytest.mark.gpu
def test_tight_table(ctx):
    from registrar_b200 import synth
    paths = _run(ctx, synth.generate("config3", n=100_000, seed=4))
    ctx.set_option("mkdirp_tight_table", 1)
    try:
        check_set(ctx, paths)
        check_set(ctx, _run(ctx, fleet(50_000, ndom=300)))
    finally:
        ctx.set_option("mkdirp_tight_table", 0)


@pytest.mark.gpu
def test_after_a_dirty_skip_batch_only_kept_records_count(ctx):
    from registrar_b200 import synth
    from registrar_b200.batch import RecordBatch
    base = synth.generate("config3", n=4000, seed=8)
    recs = [base.record(i) for i in range(base.n)]
    for i in (0, 5, 128, 1999, 3999):
        recs[i] = dict(recs[i], domain=recs[i]["domain"] + b"/x")
    batch = RecordBatch.from_records(recs, types=base.types)
    got = ctx.register_batch(batch, skip_bad=True)
    assert got.skipped.tolist() == [0, 5, 128, 1999, 3999]
    kept = batch.take(np.setdiff1d(np.arange(batch.n), got.skipped))
    from oracle import oracle
    check_set(ctx, _paths(oracle.register_batch(kept)))


@pytest.mark.gpu
def test_after_two_async_host_batches(ctx):
    from oracle import oracle
    from registrar_b200 import synth
    a, b = synth.generate("config3", n=3000, start=100), synth.generate("config5", n=2500, start=200)
    ctx.set_option("async", 1)
    try:
        ta, tb = ctx.submit(a), ctx.submit(b)
        from registrar_b200._native import RegkError
        with pytest.raises(RegkError) as e:
            ctx.mkdirp_dirs()                                   # batches in flight
        assert e.value.code == 5
        ctx.collect(ta)
        ctx.collect(tb)
    finally:
        ctx.set_option("async", 0)
    check_set(ctx, _paths(oracle.register_batch(b)))


@pytest.mark.gpu
def test_parent_dirs_result_is_untouched(ctx):
    from registrar_b200 import synth
    _run(ctx, synth.generate("config3", n=20_000, seed=12))
    raw = ctx.parent_dirs(device=True)
    n, nu = int(raw.n), int(raw.n_unique)
    before = (_dev(ctx, raw.parent_len, n, np.uint32), _dev(ctx, raw.unique_first, nu, np.uint64))
    ctx.mkdirp_dirs()
    ctx.mkdirp_requests()
    after = (_dev(ctx, raw.parent_len, n, np.uint32), _dev(ctx, raw.unique_first, nu, np.uint64))
    assert all(np.array_equal(x, y) for x, y in zip(before, after))


@pytest.mark.gpu
def test_frames_xid_wrap_flags_and_device(ctx):
    from registrar_b200 import synth
    paths = _run(ctx, synth.generate("config3", n=5000, seed=13))
    dirs, _, _ = mkdirp_set(paths)
    ctx.mkdirp_dirs()
    for xid, flags in ((1, 0), (2 ** 31 - 100, 0), (-7, 1), (2 ** 31 - 1, 2)):
        fb, fo, _ = ctx.mkdirp_requests(xid_base=xid, zk_flags=flags)
        assert fb.tobytes() == mkdirp_frames(dirs, xid, flags)
        raw = ctx.mkdirp_requests(xid_base=xid, zk_flags=flags, device=True)
        assert _dev(ctx, raw.frame_bytes, int(raw.total), np.uint8).tobytes() == fb.tobytes()
        assert np.array_equal(_dev(ctx, raw.frame_off, int(raw.n) + 1, np.uint64), fo)


@pytest.mark.gpu
def test_refusals(built):
    from registrar_b200 import _native, synth
    c = _native.Context(0)
    try:
        with pytest.raises(_native.RegkError) as e:
            c.mkdirp_requests()                                 # no set yet
        assert e.value.code == 5
        batch = synth.generate("config1")
        with pytest.raises(_native.RegkError) as e:
            c.mkdirp_dirs()                                     # no batch yet
        assert e.value.code == 5
        c.register_batch(batch, paths=False)
        with pytest.raises(_native.RegkError) as e:
            c.mkdirp_dirs()                                     # REGK_NO_PATH
        assert e.value.code == 5
        c.register_batch(batch)
        ds = c.mkdirp_dirs()
        assert ds.n == batch.n and ds.n_dirs > 0
        fb, fo, _ = c.mkdirp_requests()
        assert len(fo) == ds.n_dirs + 1
    finally:
        c.close()
