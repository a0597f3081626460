"""The walk's reply readers (regk_read_walk's two sections, its refresh level, and regk_walk_events with the path table
lookups) against walk_watch_util / walk_setwatches_util's restatements, on streams built to land on the junctions of
the chained passes: the first getChildren reply head at every phase of a span's last block (with and without frames
between the sections), payload bytes that parse as replies of section 2 or entries, stream and section lengths at span
and super-tile multiples, frontier sizes and listing counts at 2^m - 1, 2^m and 2^m + 1, levels cut inside the k-th
reply of either section or faulted at the k-th getChildren reply, random trees with mutated streams at the int32 xid
edges, the refresh level (apply, filter, two-source rebuild), near-miss notification paths at the table's growth
points, and the events reader's `start` phases and chunked feeding with the SetWatches gate closed and open.

Every case runs on three contexts in lockstep through test_walk_setwatches.Lib: a host stream, a device stream, and a
device stream with device event outputs.  Accepted: every count, the snapshot, level_off, the frontier and the zxid
high-water mark equal the model's.  Refused: REGK_ERR_INVALID_ARG naming the restatement's byte, reason, section and
node, and the read that follows gives the model's result.  CPU: the generators against the restatements alone."""
import copy
import itertools
import random
import re
import struct

import numpy as np
import pytest

import children_util as cu
import events_util as ev
import reader_fuzz_util as fz
import replies_util as ru
import setwatches_util as sw
import test_walk_setwatches as tws
import test_walk_watch as tw
import walk_setwatches_util as ws
import walk_watch_util as ww
from test_reader_fuzz import CHILDREN_REASON, EVENTS_REASON, REPLY_REASON

SESSION = ww.Driver.SESSION
wrap = ru.wrap
# frontier sizes 1, 2, 3, 2^m and 2^m + 1 up to m = 10
FS = sorted({1, 2, 3} | {2 ** m for m in range(1, 11)} | {2 ** m + 1 for m in range(1, 11)})


# ------------------------------------------------------------------------------------------------------ generators --

def rooted(f, count=None, data=None):
    """a TreeZooKeeper with f roots /r<i> (data d<i>, or data(i)), root i with i % 3 children, root 0 with `count`
    children when given -> (zk, roots)"""
    zk = ws.TreeZooKeeper()
    roots = [b"/r%06d" % i for i in range(f)]
    for i, r in enumerate(roots):
        zk.create(r, data(i) if data else b"d%d" % i, 0, False)
        for c in range(count if count is not None and i == 0 else i % 3):
            zk.create(r + b"/c%d" % c, b"", 0, False)
    return zk, roots


def section2(b, xb, f):
    """where the getChildren section starts: the end of the getData section's chain"""
    return ru.read(b, xb, f)["consumed"]


def first_listing(b, xb, f):
    """where the first getChildren reply's head sits: past the notifications and pings after the getData section"""
    pos = section2(b, xb, f)
    while fz.be32(b, pos + 4) in (ev.NOTIFY_XID, ev.PING_XID):
        pos += 4 + fz.be32(b, pos)
    return pos


def reply_index(b, xid):
    """the frame of `b` (fz.split) that carries `xid`"""
    return next(i for i, x in enumerate(fz.split(b)) if fz.be32(x, 4) == xid)


def grow(frame, extra):
    """a getData success reply with `extra` more data bytes, Stat.dataLength to match"""
    _, xid, zxid, err, d = struct.unpack_from(">iiqii", frame)
    d = max(d, 0)
    st = bytearray(frame[24 + d:])
    st[52:56] = struct.pack(">i", d + extra)
    body = struct.pack(">iqii", xid, zxid, err, d + extra) + frame[24:24 + d] + b"~" * extra + bytes(st)
    return struct.pack(">i", len(body)) + body


def place_section2(b, xb, f, target, between):
    """the level's stream with its first getChildren reply head moved to byte `target`: by a notification between the
    sections (between=True), or by growing the getData section's last success reply (between=False)"""
    at = section2(b, xb, f)
    if between:
        out = b[:at] + fz.pad_to(at, target) + b[at:]
    else:
        fr = fz.split(b[:at])
        i = max(i for i, x in enumerate(fr) if len(x) >= 88 and fz.be32(x, 4) != ev.NOTIFY_XID and fz.be32(x, 16) == 0)
        fr[i] = grow(fr[i], target - at)
        out = b"".join(fr) + b[at:]
    assert first_listing(out, xb, f) == target
    return out


DECOY_AT = 32               # where decoy_data's getChildren reply starts: past the notification's head


def decoy_data(xb, f, k):
    """node k's data: a notification whose path holds a getChildren reply for a real section-2 xid (entries inside),
    a ping, a getData reply for a section-1 xid and a notification for a root"""
    inner = cu.success(wrap(xb + f + (k * 7) % f), [b"a", b"bb", b"c%d" % k]) + ru.ping() + \
        ru.success(wrap(xb + k % f), b"x") + ev.notification(b"/r%06d" % k)
    return fz.decoy(inner)


def partial_streams(b, xb, f):
    """(what, stream) for the level's stream cut inside getData reply k and inside getChildren reply k, and with
    getChildren reply k faulted (an out-of-order xid over a listing with a bad name, a bad name, a count its frame is
    too short for), k in {0, 1, f - 1}"""
    fr = fz.split(b)
    off = [0] + list(itertools.accumulate(len(x) for x in fr))
    out = []
    for k in sorted({0, 1, f - 1} & set(range(f))):
        for sec, xid in (("getData", wrap(xb + k)), ("getChildren", wrap(xb + f + k))):
            i = reply_index(b, xid)
            for c in (1, len(fr[i]) // 2, len(fr[i]) - 1):
                out.append(("cut %s %d at %d" % (sec, k, c), b[:off[i] + c]))
        i = reply_index(b, wrap(xb + f + k))
        other = wrap(xb + f + (k + 1 if k + 1 < f else k - 1 if k else f))
        short = bytearray(cu.success(wrap(xb + f + k), [b"a"]))
        short[20:24] = struct.pack(">i", 2)
        for what, x in (("order", cu.success(other, [b"n", b"a/b"])),
                        ("name", cu.success(wrap(xb + f + k), [b"ok", b".."])), ("count", bytes(short))):
            out.append(("fault getChildren %d: %s" % (k, what), b"".join(fr[:i] + [x] + fr[i + 1:])))
    return out


def xid_base(which, f, rng):
    """a level's xid base near -2^31, near 0, or near 2^31 - 2f (never covering -1 or -2)"""
    return [-2 ** 31 + rng.randrange(3), rng.randrange(3), 2 ** 31 - 2 * f - rng.randrange(3)][which]


def near_misses(paths, held, rng):
    """notification paths that are not in `held` (the snapshot's paths) but sit next to one of `paths`: the last byte
    changed, a byte dropped, a byte or a '/' added, and every proper prefix (most of them prefixes of many paths)"""
    held, out = set(held), []
    for p in paths:
        i = rng.randrange(1, len(p))
        for q in [p[:-1] + bytes([p[-1] ^ 1]), p[:i] + p[i + 1:], p[:i] + b"x" + p[i:], p + b"/", p + b"0"] + \
                [p[:k] for k in range(1, len(p))]:
            if q not in held and q not in out:
                out.append(q)
    return out


def model_level(zk, roots, xb):
    """a fresh model with the first level framed, and the server's honest stream for it"""
    m = ws.Model()
    m.start(roots)
    return m, zk.serve(m.requests(xb, True), SESSION)


# ------------------------------------------------------------------------------------------------------------ CPU --

def test_generators_against_the_restatements():
    rng = random.Random(1)
    xb = 77
    zk, roots = rooted(3)
    m, b = model_level(zk, roots, xb)
    assert copy.deepcopy(m).read(b)["n_found"] == 3                     # the unmutated stream is accepted
    for s in (1, 2, 64):                                                         # the planted head phase and section
        for ph in range(16):
            for between in (False, True):
                t = s * fz.SPAN - 16 + ph
                p = place_section2(b, xb, 3, t, between)
                assert first_listing(p, xb, 3) == t and t in fz.cands(lambda x, q: cu.plausible(x, q, xb + 3, 3), p)
                assert copy.deepcopy(m).read(p)["n_found"] == 3
    for base in (fz.SPAN, 2 * fz.SPAN, fz.SUPER_BYTES, 2 * fz.SUPER_BYTES):
        for o in (-1, 0, 1):
            assert first_listing(place_section2(b, xb, 3, base + o, False), xb, 3) == base + o
    for f in (1, 3, 17):                                                         # decoys are section-2 candidates
        zk, roots = rooted(f, data=lambda i: decoy_data(xb, f, i))
        m, b = model_level(zk, roots, xb)
        assert copy.deepcopy(m).read(b)["n_found"] == f
        c = fz.cands(lambda x, q: cu.plausible(x, q, wrap(xb + f), f), b)
        for k in range(f):
            at = b.index(decoy_data(xb, f, k)) + DECOY_AT
            assert at in c and at < section2(b, xb, f)
    for i, f in enumerate(FS):                                                   # frontier and listing sizes
        count = 2 ** (1 + i % 10) + i % 3 - 1
        zk, roots = rooted(f, count)
        m, b = model_level(zk, roots, xb)
        assert len(m.frontier) == f
        r = cu.read(b, wrap(xb + f), f, section2(b, xb, f))
        assert max(len(n) for n in r["names"]) == count
    zk, roots = rooted(5)
    m, b = model_level(zk, roots, xb)
    kinds = set()
    for what, p in partial_streams(b, xb, 5):                                    # every partial level is refused
        with pytest.raises(ru.Refused) as e:
            copy.deepcopy(m).read(p)
        kinds.add((what.split()[0], e.value.k))
    assert kinds == {(w, k) for w in ("cut", "fault") for k in (0, 1, 4)}
    held = roots + [r + b"/c0" for r in roots]
    assert all(q not in held for q in near_misses(roots, held, rng))
    for seed in REFRESH_SEEDS:                                                   # every refresh level has a frontier
        d, b, xb = refreshed(None, seed)
        f = len(d.model.frontier)
        assert f and d.model.fnode and copy.deepcopy(d.model).read(b)
        place_section2(b, xb, f, fz.SPAN - 16, False)
        assert len(partial_streams(b, xb, f)) == 9 * len({0, 1, f - 1})


# --------------------------------------------------------------------------------------------------------- checks --

class Route:
    """an rng for tw.Lib that always takes one route: below 0.5 a device stream, below 0.3 also device event outputs"""

    def __init__(self, v):
        self.v = v

    def random(self):
        return self.v


ROUTES = (0.9, 0.4, 0.0)        # host stream and outputs; device stream; device stream and device event outputs


class Fan:
    """the walk on one context per route, each checked by test_walk_setwatches.Lib against the model"""

    def __init__(self, ctxs):
        self.libs = [tws.Lib(c, Route(v)) for c, v in zip(ctxs, ROUTES)]

    def start(self, roots):
        for lib in self.libs:
            lib.start(roots)

    def requests(self, xid, watch, frames):
        for lib in self.libs:
            lib.requests(xid, watch, frames)

    def read(self, stream, want, model):
        for lib in self.libs:
            lib.read(stream, want, model)

    def events(self, stream, start, xid_base, n_xids, want):
        for lib in self.libs:
            lib.events(stream, start, xid_base, n_xids, want)

    def refresh(self, want, model):
        for lib in self.libs:
            lib.refresh(want, model)

    def setwatches(self, max_frame, want):
        for lib in self.libs:
            lib.setwatches(max_frame, want)


def _stream(lib, b):
    return tw._cuda(b) if lib.rng.random() < 0.5 else np.frombuffer(b, np.uint8)


MSG = re.compile(r": byte (\d+): (.*)")
NODE = re.compile(r"the (getData|getChildren) reply to node (\d+) \(xid")


def _reason(text, reasons):
    got = [t for t in reasons if text.startswith(t)]
    return max(got, key=len) if got else text


def read_refusal(b, xb, f):
    """the restatement's refusal of a level's stream as (section, byte, reason, node), or None"""
    try:
        r1 = ru.read(b, xb, f)
    except ru.Refused as e:
        return ("getData", e.pos, REPLY_REASON[e.code], e.k)
    try:
        cu.read(b, wrap(xb + f), f, start=r1["consumed"])
    except cu.Refused as e:
        return ("getChildren", e.pos, CHILDREN_REASON[e.code], e.k)
    return None


def expect_refusal(d, b):
    """every context refuses regk_read_walk of `b` as the restatement does (the caller reads the level afterwards)"""
    from registrar_b200 import _native
    want = read_refusal(b, d.model.xid, len(d.model.frontier))
    assert want is not None
    for lib in d.lib.libs:
        with pytest.raises(_native.RegkError) as e:
            lib.ctx.read_walk(_stream(lib, b))
        msg = e.value.message
        m, n = MSG.search(msg), NODE.search(msg)
        assert e.value.code == _native.REGK_ERR_INVALID_ARG and m and n, msg
        reasons = (REPLY_REASON if n.group(1) == "getData" else CHILDREN_REASON).values()
        assert (n.group(1), int(m.group(1)), _reason(m.group(2), reasons), int(n.group(2))) == want, (msg, want)


def accept(d, b):
    want = d.model.read(b)
    d.lib.read(b, want, d.model)
    return want


def read_case(d, b, after):
    """`b` read as the restatement reads it: accepted, or refused and then `after` accepted -> True when `b` was"""
    if read_refusal(b, d.model.xid, len(d.model.frontier)) is None:
        accept(d, b)
        return True
    expect_refusal(d, b)
    accept(d, after)
    return False


def events_case(d, b, start, xb, nx):
    """regk_walk_events of `b` from `start` on every context as the restatement reads it -> the model's result, or
    None when both refuse (the same byte and reason; nothing marked)"""
    from registrar_b200 import _native
    try:
        want = d.model.events(b, start, xb, nx)
    except ev.Refused as e:
        for lib in d.lib.libs:
            with pytest.raises(_native.RegkError) as x:
                lib.ctx.walk_events(_stream(lib, b), start, xb, nx)
            m = MSG.search(x.value.message)
            assert x.value.code == _native.REGK_ERR_INVALID_ARG and m, x.value.message
            assert (int(m.group(1)), _reason(m.group(2), EVENTS_REASON.values())) == (e.pos, EVENTS_REASON[e.code])
        return None
    d.lib.events(b, start, xb, nx, want)
    return want


def check_mark(d):
    """the zxid high-water mark as regk_walk_setwatches' relative_zxid (with its frames and counts), on every
    context"""
    d.setwatches()


def frame(d, xb):
    frames = d.model.requests(xb, True)
    d.lib.requests(xb, True, frames)
    return frames


def begin(zk, roots, lib, xb=None):
    """a watched walk of `roots` on every context; its first level framed with xids from xb -> (Driver, the server's
    stream), or no level framed when xb is None -> (Driver, None)"""
    d = ws.Driver(zk, roots, random.Random(0), lib)
    d.model.start(roots)
    lib.start(roots)
    return d, None if xb is None else zk.serve(frame(d, xb), SESSION)


REFRESH_SEEDS = [100, 101, 102, 103, 200, 201, 202] + list(range(300, 306)) + [400, 401]


def refreshed(ctxs, seed):
    """a watched walk of a random tree, churn (with data of 0 .. 40 bytes), its events and walk_refresh; the refresh
    level framed with xids from 1000 -> (Driver, the server's stream for it)"""
    rng = random.Random(seed)
    zk = ws.TreeZooKeeper()
    ww.build_tree(zk, rng, b"/z", 3, (1, 2, 4))
    d = ws.Driver(zk, [b"/z"], rng, Fan(ctxs) if ctxs else None)
    d.start()
    mut = ww.Mutator(zk, [b"/z"], rng)
    mut.some(6)
    nodes = sorted(p for p in zk.nodes if p.startswith(b"/z"))
    for p in rng.sample(nodes, min(4, len(nodes))):
        zk.set_data(p, bytes(rng.randrange(97, 123) for _ in range(rng.randrange(41))))
    d.feed(zk.take_events(SESSION))
    d.refresh_framed()
    xb = 1000
    frames = frame(d, xb) if ctxs else d.model.requests(xb, True)
    return d, zk.serve(frames, SESSION), xb


# ------------------------------------------------------------------------------------------------------------ GPU --

@pytest.fixture(scope="module")
def ctxs(built):
    from registrar_b200 import _native
    cs = [_native.Context(0) for _ in ROUTES]
    yield cs
    for c in cs:
        c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("between", [False, True])
def test_section_boundary(ctxs, between):
    """case 1: the first getChildren reply head at every phase of the last block of span 1, 2 and 64; accepted, and cut
    1 .. 24 bytes past that head"""
    zk, roots = rooted(3)
    fan, xb = Fan(ctxs), 11
    cuts = itertools.cycle(range(1, 25))
    for s in (1, 2, 64):
        for ph in range(16):
            t = s * fz.SPAN - 16 + ph
            d, honest = begin(zk, roots, fan, xb)
            b = place_section2(honest, xb, 3, t, between)
            read_case(d, b[:t + next(cuts)], b)
            check_mark(d)


@pytest.mark.gpu
def test_payload_decoys(ctxs):
    """case 2: getData payloads holding a getChildren reply for a real section-2 xid (with entries), a ping, a getData
    reply and a notification; the chains must not start on them"""
    fan, xb = Fan(ctxs), 5
    for f in (1, 3, 17, 130):
        zk, roots = rooted(f, data=lambda i: decoy_data(xb, f, i))
        d, honest = begin(zk, roots, fan, xb)
        at = section2(honest, xb, f)
        read_case(d, honest[:at], honest)                                          # the getData section alone
        check_mark(d)


@pytest.mark.gpu
def test_stream_lengths(ctxs):
    """case 3: the level's stream cut to 0 .. 24 bytes; a getData section that ends at a span or super-tile multiple
    - 1, + 0, + 1, read whole and cut there"""
    zk, roots = rooted(3)
    fan, xb = Fan(ctxs), 3
    for L in range(25):
        d, honest = begin(zk, roots, fan, xb)
        read_case(d, honest[:L], honest)
    for base in (fz.SPAN, 2 * fz.SPAN, fz.SUPER_BYTES, 2 * fz.SUPER_BYTES):
        for o in (-1, 0, 1):
            d, honest = begin(zk, roots, fan, xb)
            b = place_section2(honest, xb, 3, base + o, o != 0)
            read_case(d, b[:base + o], b)
            check_mark(d)


def _sizes(ctxs, f, count, xb=1):
    zk, roots = rooted(f, count)
    d, honest = begin(zk, roots, Fan(ctxs), xb)
    want = accept(d, honest)
    assert want["n_found"] == f and want["n_children"] == sum(len(zk.kids[r]) for r in roots)
    while d.model.frontier:                                                        # the listed level: f >= count
        accept(d, zk.serve(frame(d, 1), SESSION))
    check_mark(d)


@pytest.mark.gpu
def test_frontier_sizes(ctxs):
    """case 4: f = 1, 2, 3, 2^m and 2^m + 1 up to 1025, root 0 listing 2^m - 1, 2^m or 2^m + 1 entries (the entry
    chain's reach at and beside a power of two), and every such count up to 1025 on a frontier of 2"""
    for i, f in enumerate(FS):
        _sizes(ctxs, f, 2 ** (1 + i % 10) + i % 3 - 1)
    for m in range(1, 11):
        for count in (2 ** m - 1, 2 ** m, 2 ** m + 1):
            _sizes(ctxs, 2, count, xb=2 ** 31 - 4 - count)


@pytest.mark.gpu
@pytest.mark.slow
def test_frontier_size_large(ctxs):
    _sizes(ctxs, 2 ** 17 + 1, 2 ** 12 + 1)


@pytest.mark.gpu
def test_partial_levels(ctxs):
    """case 5: cut inside getData reply k and getChildren reply k, and getChildren reply k faulted, k = 0, 1, f - 1:
    the entry chain bounded by the first faulting frame, and both sections' error texts"""
    fan = Fan(ctxs)
    for f, xb in ((1, 9), (2, -2 ** 31), (5, 9), (300, 2 ** 31 - 600)):
        zk, roots = rooted(f)
        d, honest = begin(zk, roots, fan, xb)
        for _, b in partial_streams(honest, xb, f):
            expect_refusal(d, b)
        accept(d, honest)
        check_mark(d)


def random_levels(ctxs, seed, tries=4):
    """case 6: random trees walked three times (xid bases near -2^31, 0 and 2^31 - 2f); per level up to `tries`
    streams with 0 .. 3 mutations from byte 0 or from the getChildren section: each refused one checked, the first
    accepted one read (else the honest stream)"""
    rng = random.Random(7000 + seed)
    zk = ws.TreeZooKeeper()
    ww.build_tree(zk, rng, b"/z", rng.choice([2, 3, 4]), (0, 1, 2, 4, 9))
    fan = Fan(ctxs)
    for which in range(3):
        d, _ = begin(zk, [b"/z"], fan)
        while d.model.frontier:
            f = len(d.model.frontier)
            xb = xid_base(which, f, rng)
            honest = zk.serve(frame(d, xb), SESSION)
            at = section2(honest, xb, f)
            for _ in range(tries):
                b, _ = fz.mutate(honest, rng, 3, rng.choice([0, at]))
                if read_refusal(b, xb, f) is None:
                    accept(d, b)
                    break
                expect_refusal(d, b)
            else:
                accept(d, honest)
        check_mark(d)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(4))
def test_random_and_mutated_levels(ctxs, seed):
    random_levels(ctxs, seed)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("seed", range(4, 24))
def test_random_and_mutated_levels_sweep(ctxs, seed):
    random_levels(ctxs, seed, tries=8)


@pytest.mark.gpu
def test_refresh_level(ctxs):
    """case 7: the refresh level (apply, filter, two-source rebuild) with its first getChildren head at every phase of
    span 1's last block; cut and faulted at reply k of either section; getData errors other than NONODE on replaced
    nodes; replaced data at every phase of a 16-byte block; mutated"""
    rng = random.Random(17)
    cuts = itertools.cycle(range(1, 25))
    for ph in range(16):
        d, honest, xb = refreshed(ctxs, 100 + ph % 4)
        f = len(d.model.frontier)
        b = place_section2(honest, xb, f, fz.SPAN - 16 + ph, ph % 2 == 1)
        t = first_listing(b, xb, f)
        expect_refusal(d, b[:t + next(cuts)])
        for _, p in partial_streams(honest, xb, f) if ph < 4 else ():
            expect_refusal(d, p)
        assert read_case(d, b, b)
        check_mark(d)
    for ph in range(16):                                       # the replaced data at phase (ph + 56) % 16 of its block
        d, honest, xb = refreshed(ctxs, 200 + ph % 3)
        f = len(d.model.frontier)
        b = fz.notification_of_len(32 + ph) + honest
        if ph % 4 == 1:                                        # a getData error on a replaced node
            fr = fz.split(b)
            i = reply_index(b, wrap(xb + rng.randrange(f)))
            fr[i] = ru.error(fz.be32(fr[i], 4), rng.choice([-4, -102, -7, -110]))
            b = b"".join(fr)
        assert read_case(d, b, b)
        d.levels()
        check_mark(d)
    for seed in range(6):
        d, honest, xb = refreshed(ctxs, 300 + seed)
        f = len(d.model.frontier)
        for _ in range(6):
            b, _ = fz.mutate(honest, rng, 3, rng.choice([0, section2(honest, xb, f)]))
            if read_refusal(b, xb, f) is None:
                accept(d, b)
                break
            expect_refusal(d, b)
        else:
            accept(d, honest)
        check_mark(d)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [511, 512, 513, 1024, 1025])
def test_table_lookups(ctxs, m):
    """case 8: a snapshot of m nodes (the table grows past 512 and 1024 nodes; 512 and 1024 fill it to its maximum
    load) built over three levels; notifications naming near misses of snapshot paths, removed nodes, and NodeDeleted
    whose parent is a root, is removed, or was never walked"""
    rng = random.Random(m)
    zk = ws.TreeZooKeeper()
    zk.create(b"/w", b"", 0, False)
    roots = [b"/t", b"/u", b"/w/r"]
    for r in roots:
        zk.create(r, b"", 0, False)
    for k in range(4):
        zk.create(b"/t/d%d" % k, b"", 0, False)
    for i in range(m - 7):
        zk.create((b"/t/d%d/n%d" % (i % 4, i)) if i % 3 else b"/u/c%d" % i, b"", 0, False)
    d = ws.Driver(zk, roots, rng, Fan(ctxs))
    d.start()
    assert len(d.model.nodes) == m
    paths = [n[0] for n in d.model.nodes]
    gone_dir, gone = b"/t/d1", rng.choice([p for p in paths if p.startswith(b"/t/d2/")])
    d.feed(ev.notification(gone_dir, ev.DELETED) + ev.notification(gone, ev.DELETED))
    assert d.model.counts()[1] == 2
    under_gone = [p for p in paths if p.startswith(gone_dir + b"/")]
    near = near_misses(rng.sample(paths, 40) + roots, paths, rng)
    names = near + [gone, gone_dir] + under_gone[:5]
    names += [b"/t/d0", b"/t/d3", b"/u", b"/w/r", b"/w", b"/"]
    notes = [ev.notification(p, rng.choice([ev.CREATED, ev.DELETED, ev.DATA_CHANGED, ev.CHILDREN_CHANGED]))
             for p in names]
    notes += [ev.notification(p, ev.DELETED) for p in (b"/t/d0", b"/u/c3", b"/w/r") + tuple(under_gone[5:8])]
    rng.shuffle(notes)
    want = events_case(d, b"".join(notes), 0, 0, 0)
    assert want["n_unmatched"] >= len(near)
    d.refresh()
    check_mark(d)


@pytest.mark.gpu
@pytest.mark.parametrize("gate", [False, True])
def test_events_stream_edges(ctxs, gate):
    """case 9: a refresh level's reply stream with mutations landing in flight (its notifications interleaved), plus
    pings, notifications and (gate open) SetWatches replies: every `start` phase after a front that chains elsewhere,
    cut 9 bytes past `start`, random chunks, and mutated"""
    rng = random.Random(21 + gate)
    d, _, _ = refreshed(ctxs, 400 + gate)
    if gate:
        check_mark(d)                                          # regk_walk_setwatches opens the gate
    mut = ww.Mutator(d.zk, [b"/z"], rng)
    f = len(d.model.frontier)
    xb = 5000
    stream = d.zk.serve(frame(d, xb), SESSION, mut.in_flight(0.4))
    accept(d, stream)
    paths = [n[0] for n in d.model.nodes]
    extras = fz.noise(rng, paths, 12) + ([sw.reply(d.zk.zxid + k) for k in range(3)] if gate else [])
    b = b"".join(fz.interleave(fz.split(stream), rng, extras))
    nx = 2 * f
    for start in list(range(16)) + [16 * rng.randrange(2, 40) + ph for ph in range(16)] + [fz.SPAN, fz.SPAN + 1]:
        s = fz.long_front(start, rng) + b
        events_case(d, s, start, xb, nx)
        events_case(d, s[:start + 9], start, xb, nx)
    events_case(d, b, len(b), xb, nx)
    for _ in range(3):                                          # chunks carrying the bytes from `consumed`
        whole = copy.deepcopy(d.model).events(b, 0, xb, nx)
        carry, fed, pos = b"", 0, []
        while fed < len(b):
            k = min(len(b), fed + rng.choice([1, 7, 20, 33, 100, 2048]))
            piece = carry + b[fed:k]
            got = events_case(d, piece, 0, xb, nx)
            pos += [fed - len(carry) + e[0] for e in got["events"]]
            carry, fed = piece[got["consumed"]:], k
        assert not carry and pos == [e[0] for e in whole["events"]]
    for _ in range(12):
        events_case(d, fz.mutate(b, rng, 3)[0], 0, xb, nx)
    check_mark(d)
