"""The registry walk on the GPU (regk_walk_start / regk_walk_requests / regk_read_walk), bit for bit against the
restatement in walk_util: snapshot paths, data, versions, owners, level_off and every count, level by level.  The
README tree; random trees of depth 1 to 8 with fan-outs from 0 to thousands; host and device streams and frames; every
race and error knob; a refused stream read again once corrected; the state rules; read_replies, read_children and
resolve results taken before a walk, unchanged after it; walk -> resolve -> answer_dns against resolve -> answer_dns on a
host snapshot of the same nodes; a million nodes under a thousand service records."""
import random

import numpy as np
import pytest

import children_util as cu
import dns_util as du
import replies_util as ru
import resolve_util as rv
import walk_util as wu
from test_resolve import compare, raw_to_dict
from test_resolve_cpu import host, service
from test_walk_cpu import AUTH

pytestmark = pytest.mark.gpu
ZK_GETDATA, ZK_GETCHILDREN = 4, 8


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def _cuda(b):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(b), np.uint8).copy()).cuda()


def frames_of(ctx, xid, device):
    if not device:
        return ctx.walk_requests(xid)[0]
    out = ctx.walk_requests(xid, device=True)
    return ctx._d2h(out.frame_bytes, int(out.total), np.uint8)


def check_level(w, want):
    for k in ("n_found", "n_missing", "n_error", "n_listed", "n_list_missing", "n_list_error", "n_children", "n_skipped",
              "consumed"):
        assert getattr(w, k) == want[k], k
    assert w.n_frontier == len(want["frontier"])


def check_snapshot(w, nodes, off):
    s = w.snapshot()
    assert w.m == len(nodes) and w.level_off.tolist() == off
    pb, jb = s.path_bytes.tobytes(), s.json_bytes.tobytes()
    po, jo = s.path_off.tolist(), s.json_off.tolist()
    assert [pb[po[j]:po[j + 1]] for j in range(w.m)] == [n[0] for n in nodes]
    assert [jb[jo[j]:jo[j + 1]] for j in range(w.m)] == [n[1] for n in nodes]
    assert s.version.tolist() == [n[2] for n in nodes] and s.owner.tolist() == [n[3] for n in nodes]
    assert (po[-1], jo[-1]) == (int(w._out.snapshot.path_total), int(w._out.snapshot.json_total))


def run(ctx, tree, roots, rng=None, xid_base=1, dev_in=False, dev_frames=False, knobs=None, before=None):
    """the walk level by level, each level against walk_util.read_level; returns (last Walk, nodes, level_off)"""
    ctx.walk_start(roots)
    nodes, off, frontier, xid, level, w = [], [0], list(roots), xid_base, 0, None
    while frontier:
        if before:
            before(tree, level, frontier)
        if any((r - xid) % 2 ** 32 < 2 * len(frontier) for r in (2 ** 32 - 1, 2 ** 32 - 2)):
            xid = 0
        fb = frames_of(ctx, xid, dev_frames)
        assert wu.parse_requests(fb, xid) == frontier
        stream = wu.answer(tree, fb, xid, rng, **(knobs(level, frontier) if knobs else {}))
        want = wu.read_level(stream, frontier, xid)
        w = ctx.read_walk(_cuda(stream) if dev_in else np.frombuffer(stream, np.uint8))
        check_level(w, want)
        nodes += want["nodes"]
        off.append(len(nodes))
        assert w.level == level + 1 and w.level_off.tolist() == off
        frontier, xid, level = want["frontier"], (xid + 2 * len(frontier)) % 2 ** 32, level + 1
    check_snapshot(w, nodes, off)
    return w, nodes, off


def test_readme_tree(ctx):
    t = wu.readme_tree()
    for dev_in, dev_frames in ((False, False), (True, True)):
        w, nodes, off = run(ctx, t, [b"/us/joyent"], dev_in=dev_in, dev_frames=dev_frames)
        assert (nodes, off) == wu.bfs(t, [b"/us/joyent"]) and off == [0, 1, 2, 3, 5]
    a = ctx.resolve(w, 30, 60)
    want = rv.resolve([(p, d) for p, d, _, _ in nodes], 30, 60)
    compare(a, want)
    assert sum(1 for k in a.q_kind if k == rv.SERVICE_SRV) == 1
    ctx.walk_start([AUTH])                                      # device=True: the raw regk_walk
    fb = ctx.walk_requests(3)[0]
    raw = ctx.read_walk(_cuda(wu.answer(t, fb, 3)), device=True)
    assert (raw.level, raw.m, raw.n_frontier, raw.snapshot.flags) == (1, 1, 2, 1)


def random_tree(rng, depth, fan, prefix=b"/t"):
    """a tree of `depth` levels under `prefix`, fan-outs drawn from `fan`; data mixes empty, service and host records"""
    t = wu.Tree()
    t.add(prefix, service(b"_http", b"_tcp", 80, None))
    level = [prefix]
    for d in range(depth - 1):
        nxt = []
        for p in level:
            for k in range(rng.choice(fan)):
                c = p + b"/n%d_%d" % (d, k)
                r = rng.random()
                data = b"" if r < 0.3 else host(b"redis_host", b"10.%d.%d.%d" % (d, k % 256, rng.randrange(256)),
                                                 rng.choice([None, 30]), [rng.randrange(1, 65536)]) if r < 0.8 else \
                    service(b"_s%d" % d, b"_tcp", rng.randrange(65536), 60)
                t.add(c, data, version=rng.randrange(-1, 5), owner=rng.choice([0, 0x1234567890]))
                nxt.append(c)
        level = nxt
    return t


@pytest.mark.parametrize("depth,fan", [(1, [0]), (2, [0, 3]), (3, [0, 1, 2, 40]), (5, [0, 1, 2, 3]), (8, [1, 1, 2]),
                                       (2, [3000]), (3, [0, 60, 70])])
def test_random_trees(ctx, depth, fan):
    rng = random.Random(depth * 100 + len(fan))
    t = random_tree(rng, depth, fan)
    roots = [b"/t"]
    w, nodes, off = run(ctx, t, roots, rng, xid_base=rng.randrange(1, 2 ** 31), dev_in=depth % 2 == 0,
                        dev_frames=depth % 3 == 0)
    assert (nodes, off) == wu.bfs(t, roots)
    assert w.n_frontier == 0


def test_many_roots_some_missing(ctx):
    rng = random.Random(7)
    t = random_tree(rng, 3, [0, 2, 5], prefix=b"/a")
    roots = [b"/zz", b"/a/n0_1", b"/a/n0_0", b"/missing/x"]
    w, nodes, off = run(ctx, t, roots, rng)
    assert (nodes, off) == wu.bfs(t, roots)


def test_races_and_errors(ctx):
    rng = random.Random(11)
    t = random_tree(rng, 5, [0, 2, 4])

    def before(tree, level, frontier):       # nodes deleted after being listed
        for p in frontier:
            if p in tree.nodes and rng.random() < 0.1:
                tree.remove(p)

    def between(tree, paths):               # created between getData and getChildren, or gone, or grown a child
        for p in paths:
            r = rng.random()
            if p not in tree.nodes and r < 0.5:
                tree.add(p, b"new")
                tree.add(p + b"/late", host(b"redis_host", b"10.1.1.1"))
            elif p in tree.nodes and r < 0.05:
                tree.remove(p)
            elif p in tree.nodes and r < 0.1:
                tree.add(p + b"/x%d" % rng.randrange(10 ** 9))

    def knobs(level, frontier):
        f = len(frontier)
        return dict(between=between, shuffle=True, noise=rng.randrange(0, 6), null=True,
                    gd_errors={rng.randrange(f): rng.choice([-4, -102, -7])} if f and rng.random() < 0.5 else {},
                    gc_errors={rng.randrange(f): rng.choice([-4, -101, -112])} if f and rng.random() < 0.5 else {},
                    trailing=ru.ping() if rng.random() < 0.5 else b"")
    for dev_in in (False, True):
        run(ctx, t, [b"/t"], rng, xid_base=2 ** 31 - 5, dev_in=dev_in, knobs=knobs, before=before)


def test_refused_stream_then_corrected(ctx):
    from registrar_b200 import _native
    t = random_tree(random.Random(5), 3, [3])
    ctx.walk_start([b"/t"])
    fb = ctx.walk_requests(1)[0]
    good = wu.answer(t, fb, 1)
    w0 = ctx.read_walk(np.frombuffer(good, np.uint8))
    fb = ctx.walk_requests(100)[0]
    frontier = wu.parse_requests(fb, 100)
    good = wu.answer(t, fb, 100)
    f = len(frontier)
    parts = wu.fz.split(good)
    parts[f] = cu.success(100 + f, [b"a/b"])                             # a name holding '/' in the first listing
    bads = [good[:-3],                                                   # truncated in the last getChildren reply
            ru.error(100, 0) + good,                                     # a success frame too short for a data length
            good[:4] + b"\x00\x00\x00\x63" + good[8:],                   # the first reply's xid outside the framing
            ru.notification() + ru.error(5000, -101) + good,             # an xid outside the framing after a notification
            b"".join(parts)]
    for bad in bads:
        for dev in (False, True):
            with pytest.raises(_native.RegkError, match=r"byte [0-9]+: .*the get(Data|Children) reply to node [0-9]+ "
                                                        r"\(xid -?[0-9]+\)"):
                ctx.read_walk(_cuda(bad) if dev else np.frombuffer(bad, np.uint8))
            with pytest.raises(wu.ru.Refused):
                wu.read_level(bad, frontier, 100)
    w = ctx.read_walk(np.frombuffer(good, np.uint8))           # nothing changed: the corrected stream reads as a clean walk
    want = wu.read_level(good, frontier, 100)
    check_level(w, want)
    assert w.level == 2 and w.m == w0.m + want["n_found"]
    ctx2 = _native.Context(0)
    try:
        w2, nodes, off = run(ctx2, t, [b"/t"])
        while w.n_frontier:
            fb = ctx.walk_requests(7)[0]
            w = ctx.read_walk(np.frombuffer(wu.answer(t, fb, 7), np.uint8))
        assert w.level_off.tolist() == off
        check_snapshot(w, nodes, off)
    finally:
        ctx2.close()


def test_state_errors_and_refusals(ctx):
    from registrar_b200 import _native
    ctx.walk_start([b"/s"])
    with pytest.raises(_native.RegkError, match="no framing"):
        ctx.read_walk(np.zeros(0, np.uint8))
    fb1 = ctx.walk_requests(1)[0]
    fb2 = ctx.walk_requests(-10)[0]                             # reframing with a new base: the last framing counts
    assert wu.parse_requests(fb1, 1) == wu.parse_requests(fb2, -10) == [b"/s"]
    t = wu.Tree()
    with pytest.raises(_native.RegkError, match="expected the getData reply to node 0 \\(xid -10\\)"):
        ctx.read_walk(np.frombuffer(wu.answer(t, fb1, 1), np.uint8))
    w = ctx.read_walk(np.frombuffer(wu.answer(t, fb2, -10), np.uint8))
    assert (w.m, w.n_missing, w.n_list_missing, w.n_frontier, w.level) == (0, 1, 1, 0, 1)
    with pytest.raises(_native.RegkError, match="complete") as e:
        ctx.walk_requests(1)
    assert e.value.code == _native.REGK_ERR_STATE
    with pytest.raises(_native.RegkError, match="no framing"):
        ctx.read_walk(np.zeros(0, np.uint8))
    ctx.walk_start([b"/a", b"/b"])
    with pytest.raises(_native.RegkError, match="cover -1"):
        ctx.walk_requests(-4)
    with pytest.raises(_native.RegkError, match="cover -2"):
        ctx.walk_requests(2 ** 32 - 5)
    ctx.walk_requests(2 ** 32 - 6)                              # [-6, -2) is fine
    for roots, msg in (([], "no roots"), ([b"/a", b"/"], "root 1 is \"/\""), ([b"a"], "root 0 is a path ZooKeeper rejects"),
                       ([b"/a/"], "root 0 is a path"), ([b""], "root 0 is a path"),
                       ([b"/x", b"/a", b"/b", b"/a"], "root 3 equals root 1"), ([b"/q", b"/a/b", b"/a"], "root 1 lies under root 2")):
        with pytest.raises(_native.RegkError, match=msg) as e:
            ctx.walk_start(roots)
        assert e.value.code == _native.REGK_ERR_INVALID_ARG
        if roots:
            assert wu.root_error(roots)[0] == int(msg.split()[1])
    assert wu.parse_requests(ctx.walk_requests(1)[0], 1) == [b"/a", b"/b"]    # a refused start changes nothing


def test_other_results_survive_a_walk(ctx):
    """read_replies, read_children and resolve results taken before a walk are byte for byte the same after it"""
    from registrar_b200 import synth
    b = synth.generate("config2", n=3000)
    got = ctx.register_batch(b)
    paths = [got.path(i) for i in range(got.n)]
    fb, _, _ = ctx.jute_requests(ZK_GETDATA, xid_base=11)
    n = got.n
    gd = ru.device_replies(got.json_bytes, got.json_off.astype(np.uint64), 11, np.arange(n, dtype=np.int32),
                           np.zeros(n, np.int64), missing=np.arange(n) % 13 == 2)
    rep = ctx.read_replies(gd)
    cfb, _, _ = ctx.children_requests(ZK_GETCHILDREN, xid_base=5000)
    dirs = [d for _, d in cu.parse_getchildren(cfb)]
    cstream = b"".join(cu.success(5000 + k, [b"x%d" % j for j in range(k % 4)]) for k in range(len(dirs)))
    ch = ctx.read_children(np.frombuffer(cstream, np.uint8))
    ans = ctx.resolve(rep, 30, 60, device=True)

    def grab():
        s = rep.snapshot()
        return (s.path_bytes.tobytes(), s.json_bytes.tobytes(), s.path_off.tobytes(), s.version.tobytes(), s.owner.tobytes(),
                ch.listing(), ctx._d2h(ch._out.listing.path_off, ch.n_children + 1, np.uint64).tobytes(),
                raw_to_dict(ctx, ans)["text"].tobytes(), raw_to_dict(ctx, ans)["sec_off"].tobytes())
    before = grab()
    run(ctx, random_tree(random.Random(1), 4, [0, 3, 9]), [b"/t"], dev_in=True)
    run(ctx, random_tree(random.Random(2), 3, [200]), [b"/t"])
    assert grab() == before
    compare(raw_to_dict(ctx, ans), rv.resolve([(paths[k], got.json(k)) for k in rep.node_rec.tolist()], 30, 60))


def dns_queries(names):
    return du.pack([du.query(n, t, ident=i) for i, n in enumerate(names) for t in (du.T_A, du.T_SRV)])


def test_walk_resolve_answer_end_to_end(ctx):
    """walk -> resolve -> answer_dns equals resolve -> answer_dns on a host snapshot of the same nodes in BFS order"""
    from registrar_b200.batch import Snapshot
    rng = random.Random(21)
    t = wu.Tree()
    t.add(b"/us")
    t.add(b"/us/zone")
    for s in range(40):
        sp = b"/us/zone/svc%d" % s
        t.add(sp, service(b"_http", b"_tcp", 8000 + s, rng.choice([None, 60])) if s % 5 else b"")
        for i in range(rng.randrange(0, 30)):
            t.add(sp + b"/i%d" % i, host(rng.choice([b"redis_host", b"host", b"moray_host"]), b"10.0.%d.%d" % (s, i),
                                         rng.choice([None, 10]), [8000 + s, 9000]))
    w = ctx.walk([b"/us"], lambda fb: wu.answer(t, fb, wu.first_xid(fb)), xid_base=2 ** 32 - 3)
    nodes, _ = wu.bfs(t, [b"/us"])
    names = [rv.name_of(p) for p, *_ in nodes] + [b"_http._tcp." + rv.name_of(p) for p, *_ in nodes] + [b"nx.zone.us"]
    msgs, off = dns_queries(names)
    a1 = ctx.resolve(w, 30, 60)
    r1 = ctx.answer_dns(msgs, off)
    a2 = ctx.resolve(Snapshot.from_nodes([(p, d) for p, d, _, _ in nodes]), 30, 60)
    r2 = ctx.answer_dns(msgs, off)
    assert a1.text.tobytes() == a2.text.tobytes() and a1.sec_off.tolist() == a2.sec_off.tolist()
    assert a1.q_kind.tolist() == a2.q_kind.tolist() and a1.q_node.tolist() == a2.q_node.tolist()
    assert r1.resp.tobytes() == r2.resp.tobytes() and r1.resp_off.tolist() == r2.resp_off.tolist()
    assert r1.n_status[du.ANSWER] > 100
    compare(a1, rv.resolve([(p, d) for p, d, _, _ in nodes], 30, 60))


@pytest.mark.slow
def test_million_nodes_under_a_thousand_services(ctx):
    """1 000 service records x 1 000 instances, host and device streams; a sampled comparison"""
    rng = random.Random(9)
    t = wu.Tree()
    t.add(b"/fleet")
    for s in range(1000):
        sp = b"/fleet/s%03d" % s
        t.add(sp, service(b"_http", b"_tcp", 80, 60))
        for i in range(1000):
            t.add(sp + b"/%06d" % i, host(b"redis_host", b"10.%d.%d.%d" % (s // 256, s % 256, i % 250), None, [6379]),
                  version=i, owner=s)
    ctx.walk_start([b"/fleet"])
    frontier, xid, w = [b"/fleet"], 1, None
    while frontier:
        fb = ctx.walk_requests(xid)[0]
        stream = wu.answer(t, fb, xid)
        w = ctx.read_walk(_cuda(stream))
        assert w.n_found == len(frontier) and w.n_error == w.n_list_error == 0
        frontier = [p + b"/" + n for p in frontier for n in t.children(p)]
        assert w.n_frontier == len(frontier)
        xid += 2 * len(frontier) if frontier else 0
    nodes, off = wu.bfs(t, [b"/fleet"])
    assert w.m == len(nodes) == 1_001_001 and w.level_off.tolist() == off
    s = w.snapshot()
    po, jo = s.path_off, s.json_off
    for j in rng.sample(range(w.m), 2000) + [0, w.m - 1]:
        assert s.path_bytes[po[j]:po[j + 1]].tobytes() == nodes[j][0]
        assert s.json_bytes[jo[j]:jo[j + 1]].tobytes() == nodes[j][1]
        assert (int(s.version[j]), int(s.owner[j])) == (nodes[j][2], nodes[j][3])
    a = ctx.resolve(w, 30, 60)
    assert sum(1 for k in a.q_kind if k == rv.SERVICE_SRV) == 1000
