"""Reconcile against node stats (regk_reconcile_owned): ephemeral owners decide REPLACE, and the repair frames carry the
versions the snapshot observed (REGK_ZK_VERSION_OBSERVED) or replace a node in one multi transaction (REGK_ZK_REPLACE).

CPU: the struct layout against the C compiler; the restatement in reconcile_owned_util against frames worked out by
hand from zookeeper.jute; the in-memory ZooKeeper model on hand cases.
GPU: every output against the restatement on host and device snapshots; the frames against the restatement; a
registry repaired end to end in the model; a node changed after the snapshot; every refusal.
"""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

import reconcile_owned_util as ou
import reconcile_util as ru
from test_reconcile import device_snapshot, drift, run, _dev, _var_host_records

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ZK_CREATE, ZK_DELETE, ZK_SETDATA, ZK_REPLACE = 1, 2, 5, 256
SESSION, OTHER, OLD = 0x1234_5678_9ABC_DEF0, 0x0FED_CBA9_8765_4321, 0x1234_5678_9ABC_DEEF
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1


# ------------------------------------------------------------------------------------------------------------ CPU --

def test_owned_struct_layout_matches_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu ", sizeof(regk_node_stat), offsetof(regk_node_stat, ephemeral_owner),
               offsetof(regk_node_stat, session), offsetof(regk_node_stat, zk_flags), offsetof(regk_node_stat, reserved),
               sizeof(regk_delta_owned));
        printf("%zu %zu %u %u %u\n", offsetof(regk_delta_owned, n_replace), offsetof(regk_delta_owned, replace),
               REGK_DELTA_REPLACE, REGK_ZK_REPLACE, REGK_ZK_VERSION_OBSERVED);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    S, D = _native.CNodeStat, _native.CDeltaOwned
    assert got == [C.sizeof(S), S.ephemeral_owner.offset, S.session.offset, S.zk_flags.offset, S.reserved.offset,
                   C.sizeof(D), D.n_replace.offset, D.replace.offset, _native.DELTA_REPLACE, _native.ZK_REPLACE,
                   _native.FLAG_ZK_VERSION_OBSERVED]
    assert "regk_reconcile_owned" in _native.EXPORTS


# one replace entry, worked out by hand from zookeeper.jute: path "/a", payload "x", version 7, zk_flags 1, xid 5
ONE_REPLACE = bytes.fromhex(
    "00000057" "00000005" "0000000e"                                          # len 87, xid 5, OpCode.multi
    "00000002" "00" "ffffffff" "00000002" "2f61" "00000007"                   # MultiHeader{delete} DeleteRequest{"/a", 7}
    "00000001" "00" "ffffffff" "00000002" "2f61" "00000001" "78"              # MultiHeader{create} CreateRequest{"/a", "x",
    "00000001" "0000001f" "00000005" "776f726c64" "00000006" "616e796f6e65"   #   [{31, world, anyone}],
    "00000001"                                                                #   EPHEMERAL}
    "ffffffff" "01" "ffffffff")                                               # MultiHeader{-1, true, -1}


def test_replace_frame_worked_out_by_hand():
    assert len(ONE_REPLACE) == 65 + 2 * 2 + 1 + 21
    assert ou.replace_frames([(b"/a", b"x", 7)], xid_base=5, group=0) == ONE_REPLACE
    assert ou.replace_frames([(b"/a", b"x", 7)], xid_base=5, group=1) == ONE_REPLACE
    # two entries in one multi: one head, the entries back to back, one close; the second version is INT32_MIN
    two = ou.replace_frames([(b"/a", b"x", 7), (b"/bc", b"", I32_MIN)], xid_base=-1, group=2, zk_flags=0)
    second = bytes.fromhex("00000002" "00" "ffffffff" "00000003" "2f6263" "80000000"
                           "00000001" "00" "ffffffff" "00000003" "2f6263" "00000000"
                           "00000001" "0000001f" "00000005" "776f726c64" "00000006" "616e796f6e65" "00000000")
    first = ONE_REPLACE[12:-9].replace(bytes.fromhex("616e796f6e6500000001"), bytes.fromhex("616e796f6e6500000000"))
    body = bytes.fromhex("ffffffff" "0000000e") + first + second + bytes.fromhex("ffffffff01ffffffff")
    assert two == len(body).to_bytes(4, "big") + body
    assert len(two) == 2 * 65 + 2 * (2 + 3) + 1 + 21
    xid, ops, multi = ou.parse_frame(two)
    assert xid == -1 and multi and [o[:2] for o in ops] == [(2, b"/a"), (1, b"/a"), (2, b"/bc"), (1, b"/bc")]
    assert ops[2][3] == I32_MIN and ops[1][2:] == (b"x", 0)


def test_versioned_frames_restatement():
    items = [(b"/a/b", b"dd", 3), (b"/a/c", b"", -1)]
    pairs = [x[:2] for x in items]
    assert ou.versioned_frames(ZK_DELETE, items, 9, 0) == (ru.frames(ZK_DELETE, pairs[:1], 9, 0, version=3) +
                                                           ru.frames(ZK_DELETE, pairs[1:], 10, 0, version=-1))
    assert ou.versioned_frames(ZK_SETDATA, [items[0]], 2 ** 31 - 1, 1) == ru.frames(ZK_SETDATA, [items[0][:2]], 2 ** 31 - 1, 1,
                                                                                   version=3)
    _, ops, multi = ou.parse_frame(ou.versioned_frames(ZK_SETDATA, items, 1, 2))
    assert multi and ops == [(5, b"/a/b", b"dd", 3), (5, b"/a/c", b"", -1)]


def test_restatement_classes():
    paths = [b"/r/a", b"/r/b", b"/r/c", b"/r/a", b"/r/d", b"/r/e"]
    pays = [b"1", b"2", b"3", b"4", b"5", b"6"]
    nodes = [(b"/r/a", b"1", 4, OTHER), (b"/r/b", b"x", 2, SESSION), (b"/r/c", b"3", 0, 0), (b"/r/q", b"", 9, SESSION),
             (b"/r/e", b"6", 1, SESSION)]
    r = ou.reconcile_owned(paths, pays, nodes, SESSION, 1)
    assert r["cls"] == [ou.REPLACE, ou.UPDATE, ou.REPLACE, ou.DUP, ou.CREATE, ou.SAME]
    assert (r["replace"], r["update"], r["delete"], r["dup"]) == ([0, 2], [1], [3], [3])
    assert (r["replace_ver"], r["update_ver"], r["delete_ver"]) == ([4, 0], [2], [9])
    assert r["obs_cls"] == [ou.KEEP, ou.KEEP, ou.KEEP, ou.DELETE, ou.KEEP]
    r = ou.reconcile_owned(paths, pays, nodes, SESSION, 0)            # persistent wanted: the ephemerals are replaced
    assert r["cls"] == [ou.REPLACE, ou.REPLACE, ou.SAME, ou.DUP, ou.CREATE, ou.REPLACE]


def test_from_nodes_takes_one_arity():
    from registrar_b200.batch import Snapshot
    s = Snapshot.from_nodes([(b"/a", b"x", 3, SESSION), (b"/b", b"", -1, 0)])
    assert s.version.tolist() == [3, -1] and s.owner.tolist() == [SESSION, 0] and s.version.dtype == np.int32
    assert Snapshot.from_nodes([(b"/a", b"x")]).version is None
    for mixed in ([(b"/a", b"x"), (b"/b", b"", 1, 0)], [(b"/a", b"x", 1, 0), (b"/b", b"")], [(b"/a", b"x", 1)]):
        with pytest.raises(ValueError):
            Snapshot.from_nodes(mixed)


def _frame(op, path, data=b"", arg=-1):
    """a single request; arg = the flags of a create, the version of a delete / setData"""
    from oracle import pyoracle
    return pyoracle.jute_request(op, path, data, 1, arg if op == 1 else 1, arg if op != 1 else -1)


def test_zookeeper_model_hand_cases():
    zk = ou.ZooKeeper()
    assert zk.create(b"/a/b", b"", SESSION) == ou.NONODE                # missing parent
    assert zk.create(b"/a", b"", SESSION, ephemeral=False) == ou.ZOK
    assert zk.create(b"/a", b"", SESSION) == ou.NODEEXISTS
    assert zk.apply_frame(_frame(1, b"/a/b", b"v", 1), SESSION) == ou.ZOK
    assert zk.nodes[b"/a/b"].owner == SESSION and zk.nodes[b"/a"].owner == 0
    assert zk.create(b"/a/b/c", b"", SESSION) == ou.NOCHILDRENFOREPHEMERALS
    assert zk.apply_frame(_frame(5, b"/a/b", b"w", 1), SESSION) == ou.BADVERSION
    assert zk.apply_frame(_frame(5, b"/a/b", b"w", 0), SESSION) == ou.ZOK
    assert zk.nodes[b"/a/b"].version == 1 and zk.nodes[b"/a/b"].data == b"w"
    assert zk.apply_frame(_frame(5, b"/a/b", b"z", -1), SESSION) == ou.ZOK and zk.nodes[b"/a/b"].version == 2
    assert zk.apply_frame(_frame(2, b"/a", b"", -1), SESSION) == ou.NOTEMPTY
    assert zk.apply_frame(_frame(2, b"/a/x", b"", -1), SESSION) == ou.NONODE
    assert zk.apply_frame(_frame(2, b"/a/b", b"", 1), SESSION) == ou.BADVERSION
    # a multi is all or nothing, each operation against the state the ones before it left
    ok = ou.replace_frames([(b"/a/b", b"new", 2)], 1, 0)
    assert zk.apply_frame(ok, OTHER) == ou.ZOK
    assert zk.nodes[b"/a/b"].data == b"new" and zk.nodes[b"/a/b"].owner == OTHER and zk.nodes[b"/a/b"].version == 0
    before = {p: (n.data, n.version, n.owner) for p, n in zk.nodes.items()}
    assert zk.create(b"/a/c", b"c", SESSION) == ou.ZOK
    bad = ou.replace_frames([(b"/a/c", b"1", 0), (b"/a/b", b"2", 5)], 1, 2)      # the second delete: BADVERSION
    assert zk.apply_frame(bad, SESSION) == ou.BADVERSION
    assert zk.nodes[b"/a/c"].data == b"c" and zk.nodes[b"/a/c"].owner == SESSION
    assert {p: (n.data, n.version, n.owner) for p, n in zk.nodes.items() if p != b"/a/c"} == before
    twice = ou.replace_frames([(b"/a/c", b"1", 0), (b"/a/c", b"2", 0)], 1, 2)    # the second delete sees version 0 again
    assert zk.apply_frame(twice, SESSION) == ou.ZOK and zk.nodes[b"/a/c"].data == b"2"
    # a persistent node with children cannot be replaced: NOTEMPTY aborts the multi
    assert zk.apply_frame(ou.replace_frames([(b"/a", b"", 0)], 1, 0), SESSION) == ou.NOTEMPTY
    assert zk.nodes[b"/a"].owner == 0


# ------------------------------------------------------------------------------------------------------------ GPU --

@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def host_snapshot(nodes):
    from registrar_b200.batch import Snapshot
    return Snapshot.from_nodes(nodes)


def device_snapshot_owned(nodes):
    import torch
    from registrar_b200.batch import Snapshot
    d = device_snapshot([(p, x) for p, x, _, _ in nodes])
    ver = torch.tensor([v for _, _, v, _ in nodes], dtype=torch.int32, device="cuda")
    own = torch.tensor([o - 2 ** 64 if o >= 2 ** 63 else o for _, _, _, o in nodes], dtype=torch.int64, device="cuda")
    return Snapshot(d.path_bytes, d.path_off, d.json_bytes, d.json_off, ver, own)


def with_stats(nodes, rng, owners=(SESSION,), frac=0.0, foreign=(OTHER,)):
    """(path, data) -> (path, data, version, owner): random versions (the extremes included), owner SESSION except a
    fraction `frac` of foreign owners"""
    vers = [0, -1, I32_MAX, I32_MIN, 1, 7]
    out = []
    for k, (p, d) in enumerate(nodes):
        v = vers[k % len(vers)] if k < 64 else rng.randrange(I32_MIN, I32_MAX + 1)
        o = rng.choice(foreign) if rng.random() < frac else owners[k % len(owners)]
        out.append((p, d, v, o))
    return out


def check_owned(ctx, paths, pays, nodes, session=SESSION, zk_flags=1, groups=(0,), frames=True):
    """reconcile_owned over host and device snapshots, host and device outputs, against the restatement; the frames"""
    from registrar_b200 import _native
    want = ou.reconcile_owned(paths, pays, nodes, session, zk_flags)
    got = ctx.reconcile_owned(host_snapshot(nodes), session, zk_flags)
    assert got.n == len(paths) and got.m == len(nodes)
    assert got.cls.tolist() == want["cls"]
    assert got.match.tolist() == want["match"]
    assert got.obs_cls.tolist() == want["obs_cls"]
    for k in ("create", "update", "dup", "delete", "replace"):
        assert getattr(got, k).tolist() == want[k], k
    assert got.n_same == want["cls"].count(ou.SAME) and got.n_replace == len(want["replace"])
    assert got.n_same + got.n_create + got.n_update + got.n_dup + got.n_replace == got.n
    raw = ctx.reconcile_owned(device_snapshot_owned(nodes), session, zk_flags, device=True)
    assert isinstance(raw, _native.CDeltaOwned) and int(raw.n_replace) == got.n_replace
    assert np.array_equal(_dev(ctx, raw.d.cls, got.n, np.uint8), got.cls)
    assert np.array_equal(_dev(ctx, raw.d.match, got.n, np.uint64), got.match)
    assert np.array_equal(_dev(ctx, raw.d.obs_cls, got.m, np.uint8), got.obs_cls)
    for k, f in (("create", "create"), ("update", "update"), ("dup", "dup"), ("delete", "del_")):
        assert np.array_equal(_dev(ctx, getattr(raw.d, f), len(getattr(got, k)), np.uint64), getattr(got, k)), k
    assert np.array_equal(_dev(ctx, raw.replace, got.n_replace, np.uint64), got.replace)
    if frames:
        check_frames(ctx, paths, pays, nodes, want, groups, zk_flags)
    return got, want


def check_frames(ctx, paths, pays, nodes, want, groups, zk_flags=1, xid=7):
    rep = [(paths[i], pays[i], v) for i, v in zip(want["replace"], want["replace_ver"])]
    upd = [(paths[i], pays[i], v) for i, v in zip(want["update"], want["update_ver"])]
    dele = [(nodes[j][0], b"", v) for j, v in zip(want["delete"], want["delete_ver"])]
    for g in groups:
        fb, fo, _ = ctx.reconcile_requests(ZK_REPLACE, xid_base=xid, group=g, zk_flags=zk_flags, observed_version=True)
        assert fb.tobytes() == ou.replace_frames(rep, xid, g, zk_flags), g
        assert int(fo[-1]) == len(fb) and len(fo) == (len(rep) + max(g, 1) - 1) // max(g, 1) + 1
        fb, _, _ = ctx.reconcile_requests(ZK_REPLACE, xid_base=xid, group=g, zk_flags=zk_flags, version=-1)
        assert fb.tobytes() == ou.replace_frames([(p, d, -1) for p, d, _ in rep], xid, g, zk_flags), g
        fb, _, _ = ctx.reconcile_requests(ZK_SETDATA, xid_base=xid, group=g, observed_version=True)
        assert fb.tobytes() == ou.versioned_frames(ZK_SETDATA, upd, xid, g), g
        fb, _, _ = ctx.reconcile_requests(ZK_DELETE, xid_base=xid, group=g, observed_version=True)
        assert fb.tobytes() == ou.versioned_frames(ZK_DELETE, dele, xid, g), g
        # without the new option the frames are regk_reconcile's
        for op, items in ((ZK_CREATE, [(paths[i], pays[i]) for i in want["create"]]), (ZK_SETDATA, [x[:2] for x in upd]),
                          (ZK_DELETE, [x[:2] for x in dele])):
            fb, _, _ = ctx.reconcile_requests(op, xid_base=xid, group=g, version=5, zk_flags=zk_flags)
            assert fb.tobytes() == ru.frames(op, items, xid, g, zk_flags=zk_flags, version=5), (op, g)


def owned_drift(paths, pays, seed, frac=0.01, foreign_frac=0.01):
    """drift() plus stats: foreign-session ephemerals (some of them with changed bytes), persistent nodes"""
    rng = random.Random(seed)
    nodes = with_stats(drift(paths, pays, seed, frac), rng, frac=foreign_frac, foreign=(OTHER, OLD, 0))
    return nodes


@pytest.mark.gpu
def test_all_owners_right_equals_reconcile(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config1"))
    nodes = with_stats(drift(paths, pays, seed=3, frac=0.02), random.Random(1))
    got, _ = check_owned(ctx, paths, pays, nodes, groups=(0, 7))
    assert got.n_replace == 0 and got.replace.size == 0
    plain = ctx.reconcile(host_snapshot(nodes))
    assert plain.n_replace == 0 and plain.replace.size == 0
    for k in ("cls", "match", "obs_cls", "create", "update", "dup", "delete"):
        assert np.array_equal(getattr(plain, k), getattr(got, k)), k
    # the plain frames equal the frames after the owned call, when no option asks for versions
    for op in (ZK_CREATE, ZK_SETDATA, ZK_DELETE):
        for g in (0, 7):
            ctx.reconcile(host_snapshot(nodes))
            a = ctx.reconcile_requests(op, xid_base=3, group=g)[0].tobytes()
            ctx.reconcile_owned(host_snapshot(nodes), SESSION)
            assert ctx.reconcile_requests(op, xid_base=3, group=g)[0].tobytes() == a


@pytest.mark.gpu
@pytest.mark.parametrize("config,n", [("config1", None), ("config3", 1_000_000)])
def test_foreign_owners(ctx, config, n):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate(config, n=n))
    nodes = owned_drift(paths, pays, seed=5)
    first = {}
    for i, p in enumerate(paths):
        first.setdefault(p, i)
    stale = [k for k, (p, d, _, _) in enumerate(nodes) if p in first and d != pays[first[p]]]
    p, d, v, _ = nodes[stale[0]]
    nodes[stale[0]] = (p, d, v, OTHER)                                  # at least one foreign node with changed bytes
    got, want = check_owned(ctx, paths, pays, nodes, groups=(0, 100) if n else (0, 1, 7, 100))
    assert got.n_replace > 0 and got.n_update > 0 and got.n_delete > 0 and got.n_create > 0
    # a foreign owner with changed bytes is REPLACE, not UPDATE
    changed = [i for i in want["replace"] if nodes[want["match"][i]][1] != pays[i]]
    assert changed


@pytest.mark.gpu
def test_persistent_and_ephemeral_wants(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=20_000, seed=3))
    nodes = list(zip(paths, pays))
    rng = random.Random(8)
    pers = with_stats(nodes, rng, owners=(SESSION, SESSION, 0))           # a third persistent: REPLACE when ephemeral is wanted
    got, _ = check_owned(ctx, paths, pays, pers, groups=(0, 7))
    assert got.n_replace == sum(1 for x in pers if x[3] == 0)
    got, _ = check_owned(ctx, paths, pays, pers, zk_flags=0, groups=(0, 7))   # persistent wanted: the ephemerals go
    assert got.n_replace == sum(1 for x in pers if x[3] != 0)


@pytest.mark.gpu
def test_dup_records_with_a_foreign_node(ctx):
    from registrar_b200.batch import RecordBatch
    recs = [{"domain": b"svc%d.example.com" % (i % 5), "hostname": b"host%d" % (i % 200), "type": b"host",
             "address": b"10.1.1.%d" % i} for i in range(300)]
    paths, pays = run(ctx, RecordBatch.from_records(recs))
    nodes = [(p, d, i, OTHER if i % 3 == 0 else SESSION) for i, (p, d) in enumerate(zip(paths[:60], pays[:60]))]
    got, want = check_owned(ctx, paths, pays, nodes, groups=(0, 7))
    assert got.n_dup == 100 and got.n_replace == 20
    assert all(got.cls[i] == ou.DUP for i in range(200, 300))
    assert got.match[200] == got.match[0]


@pytest.mark.gpu
def test_variable_hostnames_long_paths_skip_and_tight_table(ctx):
    from registrar_b200 import synth
    from registrar_b200.batch import RecordBatch
    paths, pays = run(ctx, RecordBatch.from_records(_var_host_records(20_000)))
    check_owned(ctx, paths, pays, owned_drift(paths, pays, seed=6, frac=0.05, foreign_frac=0.05), groups=(0, 7))
    doms = [b"a.b", b"c.b", b"x." * 2500 + b"y", b"x." * 2500 + b"z", b"q.r.s", b"m." * 1100 + b"n"] * 3
    recs = [{"domain": d, "hostname": b"h", "type": b"host", "address": b"1.1.1.%d" % i} for i, d in enumerate(doms)]
    paths, pays = run(ctx, RecordBatch.from_records(recs, alias=True))
    assert max(len(p) for p in paths) > 4096
    nodes = [(paths[2], pays[2], 3, OTHER), (paths[3], pays[3][:-1], I32_MAX, SESSION), (paths[5], pays[5], I32_MIN, 0),
             (paths[3][:-1], b"", -1, SESSION), (paths[2] + b"/k", b"", 0, OTHER)]
    got, _ = check_owned(ctx, paths, pays, nodes, groups=(0, 1, 7))
    assert got.n_replace == 2 and got.n_update == 1
    base = synth.generate("config3", n=4000, seed=8)
    recs = [base.record(i) for i in range(base.n)]
    for i in (0, 5, 128, 1999, 3999):
        recs[i] = dict(recs[i], domain=recs[i]["domain"] + b"/x")
    paths, pays = run(ctx, RecordBatch.from_records(recs, types=base.types), skip_bad=True)
    check_owned(ctx, paths, pays, owned_drift(paths, pays, seed=4, frac=0.05, foreign_frac=0.05), groups=(0, 7))
    ctx.set_option("reconcile_tight_table", 1)
    try:
        paths, pays = run(ctx, synth.generate("config3", n=100_000, seed=4))
        check_owned(ctx, paths, pays, owned_drift(paths, pays, seed=2, frac=0.02), groups=(0, 100))
    finally:
        ctx.set_option("reconcile_tight_table", 0)


@pytest.mark.gpu
def test_frames_with_extreme_versions_and_wrapping_xid(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=5000, seed=11))
    rng = random.Random(2)
    nodes = owned_drift(paths, pays, seed=12, frac=0.05, foreign_frac=0.05)
    nodes = [(p, d, [0, -1, I32_MAX, I32_MIN][k % 4], o) for k, (p, d, _, o) in enumerate(nodes)]
    rng.shuffle(nodes)
    _, want = check_owned(ctx, paths, pays, nodes, frames=False)
    for v in (0, -1, I32_MAX, I32_MIN):
        assert v in want["replace_ver"] and v in want["update_ver"] and v in want["delete_ver"]
    for g in (0, 1, 7, 100):
        check_frames(ctx, paths, pays, nodes, want, (g,), xid=2 ** 31 - 3)
    # frames live until the next call and survive a later batch
    rep_frames = ctx.reconcile_requests(ZK_REPLACE, xid_base=1, group=7, observed_version=True)[0].tobytes()
    ctx.register_batch(synth.generate("config1"))
    assert ctx.reconcile_requests(ZK_REPLACE, xid_base=1, group=7, observed_version=True)[0].tobytes() == rep_frames


def spilled_tiles(lens):
    """how many 64-entry tiles of a gathered stream with these entry lengths exceed the framing kernels' staging budget
    (9/8 of a tile's mean share + 1024 bytes, in 16-byte blocks) and are framed byte-wise"""
    n = len(lens)
    off = np.concatenate([[0], np.cumsum(np.asarray(lens, np.int64))])
    cap = (min(int(off[-1]) * 64 // n * 9 // 8 + 1024, 65520) + 15) // 16 * 16
    return sum(1 for r0 in range(0, n, 64)
               if ((int(off[r0]) & 15) + int(off[min(r0 + 64, n)] - off[r0]) + 15) // 16 * 16 > cap)


def fallback_case(ctx):
    """3 000 alias records, two runs of 16 with paths of about 5 KB; every fourth record SAME, drifted (UPDATE),
    foreign-owned (REPLACE) or missing with a stale sibling node (CREATE + DELETE).  Each list gets two runs of four
    long entries, so tiles of each list both fit the staging budget and exceed it.  Returns (paths, payloads, nodes)."""
    from registrar_b200.batch import RecordBatch
    long_ = lambda i: 1000 <= i < 1016 or 2000 <= i < 2016
    recs = [{"domain": (b"x." * 2500 + b"y%d" % i) if long_(i) else b"s%d.dc%d.example.com" % (i, i % 3),
             "hostname": b"h", "type": b"host", "address": b"10.2.%d.%d" % (i % 200, i % 7)} for i in range(3000)]
    paths, pays = run(ctx, RecordBatch.from_records(recs, alias=True))
    vers = [0, -1, I32_MAX, I32_MIN, 5]
    nodes = []
    for i, (p, d) in enumerate(zip(paths, pays)):
        v = vers[i % len(vers)]
        mode = i % 4
        if mode == 3:
            nodes.append((p + b"z", b"old", v, SESSION))
        else:
            nodes.append((p, d + b" " if mode == 1 else d, v, OTHER if mode == 2 else SESSION))
    return paths, pays, nodes


@pytest.mark.gpu
def test_byte_wise_framing_fallback(ctx):
    """replace, setData and delete lists of 750 entries whose long-path tiles exceed the staging budget: the byte-wise
    fallback of regk_jute_entry_kernel frames them, next to staged tiles, for single requests and for multi transactions
    that cross tiles"""
    paths, pays, nodes = fallback_case(ctx)
    got, want = check_owned(ctx, paths, pays, nodes, groups=(0, 7, 100))
    assert got.n_replace == got.n_update == got.n_delete == got.n_create == 750
    for lens in ([len(paths[i]) for i in want["replace"]], [len(paths[i]) for i in want["update"]],
                 [len(nodes[j][0]) for j in want["delete"]]):
        assert 0 < spilled_tiles(lens) < (len(lens) + 63) // 64
    assert max(len(p) for p in paths) > 5000


def _build_registry(paths, pays, rng):
    """a registry in the model built by valid operations: drifted data, missing nodes, foreign and old-session
    ephemerals, persistent nodes, arbitrary versions, nodes the batch no longer has.  Returns (zk, snapshot nodes)."""
    import mkdirp_util
    zk = ou.ZooKeeper()
    firsts = {}
    for p, d in zip(paths, pays):
        firsts.setdefault(p, d)
    leaves = {}
    for k, (p, d) in enumerate(firsts.items()):
        mode = k % 10
        if mode == 0:
            continue                                                   # missing
        owner = {1: OTHER, 2: OLD, 3: 0}.get(mode, SESSION)
        data = d if mode not in (4, 5) else d[:-1] + b"~"            # drifted data
        leaves[p] = (data, owner)
        if mode == 6:
            leaves[p + b"x"] = (b"gone", SESSION)                      # a node the batch does not have
    dirs = set()
    for p in leaves:
        for a in mkdirp_util.ancestors(mkdirp_util.dir_of(p)):
            dirs.add(a)
    for dd in sorted(dirs, key=lambda x: x.count(b"/")):
        assert zk.create(dd, b"", 0, ephemeral=False) == ou.ZOK
    for p, (data, owner) in leaves.items():
        assert zk.create(p, data, owner, ephemeral=owner != 0) == ou.ZOK
        for _ in range(rng.randrange(0, 3)):
            assert zk.set_data(p, data) == ou.ZOK                       # arbitrary versions
    return zk, dirs


def _snapshot(zk, dirs):
    return [(p, n.data, n.version, n.owner) for p, n in sorted(zk.nodes.items()) if p not in dirs]


@pytest.mark.gpu
def test_end_to_end_repair_in_the_model(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=3000, seed=21))
    zk, dirs = _build_registry(paths, pays, random.Random(4))
    nodes = _snapshot(zk, dirs)
    d, _ = check_owned(ctx, paths, pays, nodes, frames=False)
    assert d.n_create and d.n_update and d.n_delete and d.n_replace
    fb, fo, _ = ctx.reconcile_requests(ZK_DELETE, observed_version=True)
    assert set(zk.apply_frames(fb, fo, SESSION)) == {ou.ZOK}
    ctx.mkdirp_dirs()
    fb, fo, _ = ctx.mkdirp_requests(zk_flags=0)
    assert set(zk.apply_frames(fb, fo, SESSION)) <= {ou.ZOK, ou.NODEEXISTS}
    fb, fo, _ = ctx.reconcile_requests(ZK_CREATE, zk_flags=1, group=7)
    assert set(zk.apply_frames(fb, fo, SESSION)) == {ou.ZOK}
    fb, fo, _ = ctx.reconcile_requests(ZK_SETDATA, observed_version=True, group=3)
    assert set(zk.apply_frames(fb, fo, SESSION)) == {ou.ZOK}
    fb, fo, _ = ctx.reconcile_requests(ZK_REPLACE, zk_flags=1, observed_version=True, group=5)
    assert set(zk.apply_frames(fb, fo, SESSION)) == {ou.ZOK}
    want = {}
    for p, x in zip(paths, pays):
        want.setdefault(p, x)
    all_dirs = {p for p in zk.nodes if any(q.startswith(p + b"/") for q in want)}
    after = _snapshot(zk, all_dirs)
    assert {p: x for p, x, _, _ in after} == want
    assert all(o == SESSION for _, _, _, o in after)
    again = ctx.reconcile_owned(host_snapshot(after), SESSION)
    assert again.n_same == again.n - (len(paths) - len(want)) and again.n_dup == len(paths) - len(want)
    assert again.n_create == again.n_update == again.n_delete == again.n_replace == 0


@pytest.mark.gpu
def test_node_changed_after_the_snapshot(ctx):
    from registrar_b200 import synth
    paths, pays = run(ctx, synth.generate("config3", n=2000, seed=22))
    zk, dirs = _build_registry(paths, pays, random.Random(5))
    nodes = _snapshot(zk, dirs)
    d = ctx.reconcile_owned(host_snapshot(nodes), SESSION)
    upd, rep = paths[int(d.update[0])], [paths[int(i)] for i in d.replace[:6]]
    assert zk.set_data(upd, b"meanwhile") == ou.ZOK                      # another writer, after the snapshot
    assert zk.set_data(rep[3], zk.nodes[rep[3]].data) == ou.ZOK
    before = {p: (zk.nodes[p].data, zk.nodes[p].version, zk.nodes[p].owner) for p in rep}
    fb, fo, _ = ctx.reconcile_requests(ZK_SETDATA, observed_version=True)
    res = zk.apply_frames(fb, fo, SESSION)
    assert res[0] == ou.BADVERSION and set(res[1:]) <= {ou.ZOK}
    assert zk.nodes[upd].data == b"meanwhile"
    fb, fo, _ = ctx.reconcile_requests(ZK_REPLACE, observed_version=True, group=6)
    res = zk.apply_frames(fb, fo, SESSION)
    assert res[0] == ou.BADVERSION and set(res[1:]) <= {ou.ZOK}
    assert {p: (zk.nodes[p].data, zk.nodes[p].version, zk.nodes[p].owner) for p in rep} == before


@pytest.mark.gpu
def test_owned_refusals_and_untouched_results(built):
    import torch
    from registrar_b200 import _native, synth
    c = _native.Context(0)

    def refused(code, fn, text=None):
        with pytest.raises(_native.RegkError) as e:
            fn()
        assert e.value.code == code, e.value.message
        if text:
            assert text in e.value.message, e.value.message

    try:
        paths, pays = run(c, synth.generate("config3", n=20_000, seed=12))
        nodes = owned_drift(paths, pays, seed=6, foreign_frac=0.05)
        snap = host_snapshot(nodes)
        raw = c.parent_dirs(device=True)
        n, nu = int(raw.n), int(raw.n_unique)
        before = (_dev(c, raw.parent_len, n, np.uint32), _dev(c, raw.unique_first, nu, np.uint64))
        dirs = c.mkdirp_dirs().dirs()
        frames = c.jute_requests(ZK_SETDATA, group=7)[0].tobytes()
        plain = c.reconcile(snap)
        plain_frames = c.reconcile_requests(ZK_SETDATA, group=7)[0].tobytes()
        for op in (ZK_REPLACE, ZK_SETDATA, ZK_DELETE):                 # after a plain reconcile: REGK_ERR_STATE
            refused(5, lambda: c.reconcile_requests(op, observed_version=op != ZK_REPLACE), "reconcile_owned")
        check_owned(c, paths, pays, nodes, frames=False)
        refused(1, lambda: c.reconcile_requests(ZK_CREATE, observed_version=True))
        refused(1, lambda: c.reconcile_requests(ZK_REPLACE, group=32769))
        assert c.reconcile_requests(ZK_REPLACE, group=32768)[1].size == 2
        refused(1, lambda: c.reconcile_requests(257))
        after = (_dev(c, raw.parent_len, n, np.uint32), _dev(c, raw.unique_first, nu, np.uint64))
        assert all(np.array_equal(x, y) for x, y in zip(before, after))
        assert c.mkdirp_dirs().dirs() == dirs
        assert c.jute_requests(ZK_SETDATA, group=7)[0].tobytes() == frames
        again = c.reconcile(snap)
        for k in ("cls", "match", "obs_cls", "create", "update", "dup", "delete"):
            assert np.array_equal(getattr(plain, k), getattr(again, k)), k
        assert c.reconcile_requests(ZK_SETDATA, group=7)[0].tobytes() == plain_frames
        # the stat refusals
        cin, keep = snap.cdecode_in()
        st, skeep = snap.cnode_stat(SESSION, 1)

        def owned(stat, zk_flags=None, session=None):
            s = _native.CNodeStat(stat.version, stat.ephemeral_owner, stat.session if session is None else session,
                                  stat.zk_flags if zk_flags is None else zk_flags, 0)
            return c._lib.regk_reconcile_owned(c._h, C.byref(cin), C.byref(s), 0, C.byref(_native.CDeltaOwned()))
        assert owned(st) == 0
        assert c._lib.regk_reconcile_owned(c._h, C.byref(cin), None, 0, C.byref(_native.CDeltaOwned())) == 1
        refused(5, lambda: c.reconcile_requests(ZK_CREATE))            # a refused call leaves no result
        for bad in (2, 3, 4, 8, 16):
            assert owned(st, zk_flags=bad) == 1
        assert owned(st, session=0) == 1
        assert owned(st, zk_flags=0, session=0) == 0                   # persistent: no session needed
        assert owned(_native.CNodeStat(None, st.ephemeral_owner, SESSION, 1, 0)) == 1
        assert owned(_native.CNodeStat(st.version, None, SESSION, 1, 0)) == 1
        # the CreateMode of the creates and replaces must be the one the reconcile classified with
        c.reconcile_owned(snap, SESSION, zk_flags=0)
        refused(1, lambda: c.reconcile_requests(ZK_REPLACE, zk_flags=1), "CreateMode")
        refused(1, lambda: c.reconcile_requests(ZK_CREATE, zk_flags=1), "CreateMode")
        c.reconcile_requests(ZK_REPLACE, zk_flags=0)
        c.reconcile_requests(ZK_CREATE, zk_flags=0)
        c.reconcile_requests(ZK_DELETE, zk_flags=1)                    # no CreateMode in a delete
        # device stats: misaligned pointers are refused by the library
        dev = device_snapshot_owned(nodes[:1000])
        from registrar_b200.batch import Snapshot
        dcin, dkeep = dev.cdecode_in()
        dst, dskeep = dev.cnode_stat(SESSION, 1)
        for ver, own in ((dst.version + 2, dst.ephemeral_owner), (dst.version, dst.ephemeral_owner + 4)):
            s = _native.CNodeStat(ver, own, SESSION, 1, 0)
            assert c._lib.regk_reconcile_owned(c._h, C.byref(dcin), C.byref(s), 0, C.byref(_native.CDeltaOwned())) == 1
            assert "misaligned" in c._lib.regk_last_error(c._h).decode()
        d = c.reconcile_owned(dev, SESSION)
        assert d.m == 1000
        # the Python layer refuses what the library cannot see: missing, short or mistyped stats
        bad = [(None, dev.owner), (dev.version[:999], dev.owner), (dev.version, dev.owner[:999]),
               (dev.version.to(torch.int64), dev.owner), (dev.version, dev.owner.to(torch.int32)),
               (dev.version.view(torch.uint8), dev.owner)]
        for ver, own in bad:
            with pytest.raises(ValueError):
                c.reconcile_owned(Snapshot(dev.path_bytes, dev.path_off, dev.json_bytes, dev.json_off, ver, own), SESSION)
        hs = host_snapshot(nodes[:10])
        for ver, own in ((hs.version[:9], hs.owner), (hs.version, hs.owner[:9]),
                         (hs.version.astype(np.float64), hs.owner), (hs.version.astype(np.int64) + 2 ** 31, hs.owner)):
            with pytest.raises(ValueError):
                c.reconcile_owned(Snapshot(hs.path_bytes, hs.path_off, hs.json_bytes, hs.json_off, ver, own), SESSION)
    finally:
        c.close()
