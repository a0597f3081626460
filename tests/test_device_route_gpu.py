"""The device-resident route (REGK_IN_DEVICE | REGK_OUT_DEVICE) as a caller that keeps its batches on the GPU drives
it, against the oracle byte for byte, offsets included.

Every input array lives in its own exact-size regk_dev_alloc allocation with *_len equal to the data's end: a caching
allocator's rounded-up blocks would hide a read past the caller's array (compute-sanitizer's memcheck sees it here, see
sanitize_device_types_run.py).  The queue tests run the context on a torch stream with option "async" = 1: batches
rotate through the four workspaces that a side stream re-zeroes, the device outputs are single-buffered, so each
batch's streams are copied away in stream order right behind its kernels and compared once the queue has drained."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle
from registrar_b200 import synth
from registrar_b200._native import REGK_ERR_STATE, OutOfDomainError, RegkError, _as_np, _offsets, host_cbatch
from registrar_b200.batch import (BAD_DOMAIN_BYTE, FLAG_IN_DEVICE, FLAG_NO_JSON, FLAG_NO_PATH, FLAG_OUT_DEVICE,
                                  RecordBatch)

pytestmark = pytest.mark.gpu

FIELDS = ("domain_bytes", "domain_off", "host_bytes", "host_off", "type_id", "addr_bytes", "addr_off", "ttl",
          "ports_off", "ports", "ports_present")


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


class DeviceBatch:
    """A host RecordBatch in one exact-size device allocation per array; `cb` is its regk_batch (REGK_IN_DEVICE).
    An empty array is passed as NULL with length 0."""

    def __init__(self, ctx, hb, flags=0):
        self.ctx, self.ptrs = ctx, []
        cb, keep = host_cbatch(hb, flags | FLAG_IN_DEVICE)
        for f, a in zip(FIELDS, keep):
            setattr(cb, f, self._put(a))
        self.cb, self.batch = cb, hb

    def _put(self, a):
        if a is None or a.nbytes == 0:
            return None
        p = self.ctx.dev_alloc(a.nbytes)
        self.ptrs.append(p)
        self.ctx._check(self.ctx._lib.regk_memcpy_h2d(self.ctx._h, C.c_void_p(p), a.ctypes.data_as(C.c_void_p), a.nbytes))
        return p

    def close(self):
        for p in self.ptrs:
            self.ctx.dev_free(p)
        self.ptrs = []


def fetch(res, n):
    """(path_bytes, path_off, json_bytes, json_off) of a finished regk_result, device (multigpu.device_tensor) or host."""
    if res.flags & FLAG_OUT_DEVICE:
        import torch
        from registrar_b200 import multigpu
        dev = torch.device("cuda", 0)
        get = lambda p, c, dt: multigpu.device_tensor(p, c, dt, dev).cpu().numpy()
        return (get(res.path_bytes, int(res.path_total), torch.uint8), get(res.path_off, n + 1, torch.int64).view(np.uint64),
                get(res.json_bytes, int(res.json_total), torch.uint8), get(res.json_off, n + 1, torch.int64).view(np.uint64))
    return (_as_np(res.path_bytes, int(res.path_total), np.uint8).copy(), _offsets(res, "path_off", n).astype(np.uint64),
            _as_np(res.json_bytes, int(res.json_total), np.uint8).copy(), _offsets(res, "json_off", n).astype(np.uint64))


def assert_streams(got, want, paths=True, payloads=True, what=""):
    pb, po, jb, jo = got
    assert want.bad_bits == 0
    if paths:
        assert np.array_equal(po, want.path_off), "path offsets " + what
        assert np.array_equal(pb, want.path_bytes), "path bytes " + what
    if payloads:
        assert np.array_equal(jo, want.json_off), "payload offsets " + what
        assert np.array_equal(jb, want.json_bytes), "payload bytes " + what


def run_route(ctx, hb, in_dev, out_dev, flags=0):
    """One synchronous regk_register_batch of `hb` on the given route; returns (regk_result, fetched streams)."""
    ctx.set_types(hb.types)
    if in_dev:
        db = DeviceBatch(ctx, hb, flags)
        cb = db.cb
    else:
        db = None
        cb, keep = host_cbatch(hb, flags)
    if out_dev:
        cb.flags |= FLAG_OUT_DEVICE
    try:
        res = ctx.register_raw(cb)
        return res, fetch(res, hb.n)
    finally:
        if db is not None:
            db.close()


def check_route(ctx, hb, in_dev, out_dev, want=None, modes=("default", "no_path", "no_json", "force_generic")):
    want = want if want is not None else oracle.register_batch(hb)
    for mode in modes:
        flags = {"no_path": FLAG_NO_PATH, "no_json": FLAG_NO_JSON}.get(mode, 0)
        ctx.set_option("force_generic", 1 if mode == "force_generic" else 0)
        try:
            res, got = run_route(ctx, hb, in_dev, out_dev, flags)
        finally:
            ctx.set_option("force_generic", 0)
        what = "(%s, n=%d)" % (mode, hb.n)
        assert res.bad_bits == 0
        assert_streams(got, want, paths=mode != "no_path", payloads=mode != "no_json", what=what)
        if mode == "no_path":
            assert res.path_total == 0
        if mode == "no_json":
            assert res.json_total == 0
    return want


def _records_case(name):
    base = synth.generate("config3", n=700, start=4242)
    recs = [base.record(i) for i in range(base.n)]
    if name == "host_off":
        for i, r in enumerate(recs):
            r["hostname"] = b"h%x" % (i * 2654435761 % (1 << (4 + i % 50)))
    elif name == "ports_present":                       # explicit empty arrays next to absent and full ones
        for i, r in enumerate(recs):
            r["ports"] = [None, [], [80, 443], [], [65535]][i % 5]
    elif name == "empty_labels":
        for i, r in enumerate(recs):
            if i % 97 == 5:
                r["domain"] = b"a..b." + r["domain"]
    return RecordBatch.from_records(recs, types=base.types, alias=name == "alias")


def route_case(name):
    if name.startswith("n="):
        n = int(name[2:])
        return synth.generate("config3", n=n, start=1_000 + n)
    if name == "start_99999999000":
        return synth.generate("config3", n=2_000, start=99_999_999_000)
    if name == "ports_off_null":
        b = synth.generate("config1", n=600, start=3)
        b.ports_off = b.ports = None
        return b
    return _records_case(name)


ROUTE_CASES = ["n=0", "n=1", "n=127", "n=128", "n=129", "n=4097", "start_99999999000", "alias", "host_off",
               "ports_off_null", "ports_present", "empty_labels"]
ROUTES = [(True, True), (True, False), (False, True)]


@pytest.mark.parametrize("in_dev,out_dev", ROUTES, ids=["dev_in_dev_out", "dev_in_host_out", "host_in_dev_out"])
@pytest.mark.parametrize("case", ROUTE_CASES)
def test_route_matrix(ctx, case, in_dev, out_dev):
    hb = route_case(case)
    if case == "ports_off_null":
        assert hb.ports_off is None
    if case == "ports_present":
        assert hb.ports_present is not None
    check_route(ctx, hb, in_dev, out_dev)


# --- the queue ---------------------------------------------------------------------------------------------------

QUEUE_N = 150_000                   # more tiles than one wave of the compose kernels


def queue_batches():
    """12 batches of one size and different content: fixed-stride, variable-length and alias nodes, two workloads.  With
    one size every batch needs the same workspace as the batch four places before it, which left its ring entry to the
    side stream to clean, as in a benchmark loop."""
    out = []
    for i in range(12):
        b = synth.generate("config3" if i % 3 else "config1", n=QUEUE_N, start=1_000_000 * i + 7)
        if i in (4, 9):
            recs = [b.record(j) for j in range(b.n)]
            b = RecordBatch.from_records(recs, types=b.types, alias=True)
        elif i in (2, 7):
            recs = [b.record(j) for j in range(b.n)]
            for j, r in enumerate(recs):
                r["hostname"] = b"host-%d" % (j * 7919 % (10 ** (1 + j % 9)))
            b = RecordBatch.from_records(recs, types=b.types)
        out.append(b)
    return out


class Queue:
    """The context on a torch stream, "async" = 1: submit() enqueues a batch and, behind it on the same stream, copies
    of its output streams (sizes from the oracle) out of the single-buffered device outputs."""

    def __init__(self, ctx, time_every=3):
        import torch
        self.torch, self.ctx = torch, ctx
        self.dev = torch.device("cuda", 0)
        self.stream = torch.cuda.Stream(device=self.dev)
        ctx.set_stream(self.stream.cuda_stream)
        self.time_every = time_every
        self.out = None                                 # device output pointers (stable once they stop growing)

    def start(self):
        self.ctx.set_option("async", 1)
        self.ctx.set_option("time_every", self.time_every)

    def reserve(self, want):
        """Device tensors for one batch's streams (sizes from the oracle), allocated before anything is queued."""
        torch, n = self.torch, len(want.path_off) - 1
        return [torch.empty(int(want.path_off[-1]), dtype=torch.uint8, device=self.dev),
                torch.empty(n + 1, dtype=torch.int64, device=self.dev),
                torch.empty(int(want.json_off[-1]), dtype=torch.uint8, device=self.dev),
                torch.empty(n + 1, dtype=torch.int64, device=self.dev)]

    def submit(self, db, snap):
        """Enqueue a batch, then (with `snap` from reserve()) copies of its streams into `snap`."""
        from registrar_b200 import multigpu
        torch = self.torch
        res = self.ctx.register_raw(db.cb)
        if snap is not None:
            with torch.cuda.stream(self.stream):
                for dst, src, dt in zip(snap, self.out, (torch.uint8, torch.int64, torch.uint8, torch.int64)):
                    dst.copy_(multigpu.device_tensor(src, dst.numel(), dt, self.dev))
        return res, snap

    def close(self):
        self.ctx.set_option("async", 0)
        self.ctx.set_option("time_every", 1)
        self.ctx.set_own_stream()


def snap_np(snap):
    pb, po, jb, jo = [t.cpu().numpy() for t in snap]
    return pb, po.view(np.uint64), jb, jo.view(np.uint64)


def _prime(ctx, q, dbs, wants):
    """Synchronous runs of the batches that need the largest path and payload buffers, each checked against the oracle:
    the single-buffered device outputs stop growing, so the queue's copies read them where these runs left them."""
    def path_cap(b):
        return int(b.domain_off[-1]) + (0 if b.alias else len(b.host_bytes)) + 2 * b.n

    def json_cap(b):
        return 2 * int(b.addr_off[-1]) + 11 * (int(b.ports_off[-1]) if b.ports_off is not None else 0) + 77 * b.n
    clean = [k for k in range(len(dbs)) if wants[k].bad_bits == 0]
    for i in sorted({max(clean, key=lambda k: cap(dbs[k].batch)) for cap in (path_cap, json_cap)}):
        res = ctx.register_raw(dbs[i].cb)
        assert_streams(fetch(res, dbs[i].batch.n), wants[i], what="(priming run of batch %d)" % i)
    q.out = (res.path_bytes, res.path_off, res.json_bytes, res.json_off)


def test_queue_batch_by_batch(ctx):
    """12 batches of one size in flight: batches 4..11 each reuse the workspace of the batch four places before it, which
    only the side stream re-zeroed.  Every batch's totals, bad bits and generic tiles, and its streams copied away right
    behind its kernels, timed and untimed batches alike."""
    batches = queue_batches()
    ctx.set_types(batches[0].types)
    wants = [oracle.register_batch(b) for b in batches]
    dbs = [DeviceBatch(ctx, b, FLAG_OUT_DEVICE) for b in batches]
    q = Queue(ctx, time_every=3)
    try:
        _prime(ctx, q, dbs, wants)
        q.start()
        snaps = [q.reserve(w) for w in wants]
        subs = [q.submit(db, snap) for db, snap in zip(dbs, snaps)]
        results = [ctx.finish(res) for res, _ in subs]
        q.torch.cuda.synchronize()
        timed = [r.kernel_ms > 0 for r in results]
        for i, (r, (_, snap), want) in enumerate(zip(results, subs, wants)):
            assert (int(r.path_total), int(r.json_total)) == (int(want.path_off[-1]), int(want.json_off[-1])), i
            assert r.bad_bits == 0 and r.generic_tiles == 0, i
            assert (r.path_bytes, r.path_off, r.json_bytes, r.json_off) == q.out, "the outputs moved"
            assert_streams(snap_np(snap), want, what="(batch %d, %s)" % (i, "timed" if timed[i] else "untimed"))
        assert sum(timed) == 4 and all(timed[i] == timed[i + 3] for i in range(9)), timed
    finally:
        q.close()
        for db in dbs:
            db.close()


def test_queue_growing_batches(ctx):
    """Each batch larger than all before it: output buffers and workspaces are reallocated while batches are in flight."""
    batches = [synth.generate("config3", n=n, start=n) for n in (500, 1_500, 4_500, 13_500, 40_500, 121_500)]
    ctx.set_types(batches[0].types)
    wants = [oracle.register_batch(b) for b in batches]
    dbs = [DeviceBatch(ctx, b, FLAG_OUT_DEVICE) for b in batches]
    q = Queue(ctx, time_every=1)
    try:
        q.start()
        subs = [q.submit(db, None) for db in dbs]
        results = [ctx.finish(res) for res, _ in subs]
        for r, want in zip(results, wants):
            assert (int(r.path_total), int(r.json_total)) == (int(want.path_off[-1]), int(want.json_off[-1]))
            assert r.bad_bits == 0
        assert_streams(fetch(results[-1], batches[-1].n), wants[-1], what="(last batch)")
    finally:
        q.close()
        for db in dbs:
            db.close()


def test_queue_out_of_domain_batch(ctx):
    """A batch with an out-of-domain record in the middle of the queue reports its own first record; its neighbours
    are unaffected."""
    batches = queue_batches()[:7]
    recs = [batches[3].record(j) for j in range(batches[3].n)]
    bad_at = 1_234
    recs[bad_at]["domain"] = recs[bad_at]["domain"] + b"/x"
    batches[3] = RecordBatch.from_records(recs, types=batches[3].types)
    ctx.set_types(batches[0].types)
    wants = [oracle.register_batch(b) for b in batches]
    assert wants[3].bad_bits == BAD_DOMAIN_BYTE and wants[3].first_bad == bad_at
    dbs = [DeviceBatch(ctx, b, FLAG_OUT_DEVICE) for b in batches]
    q = Queue(ctx)
    try:
        _prime(ctx, q, dbs, wants)
        q.start()
        subs = [q.submit(db, None if i == 3 else q.reserve(w)) for i, (db, w) in enumerate(zip(dbs, wants))]
        for i, (res, snap) in enumerate(subs):
            if i == 3:
                with pytest.raises(OutOfDomainError) as ei:
                    ctx.finish(res)
                assert ei.value.result.bad_bits == BAD_DOMAIN_BYTE and ei.value.result.first_bad == bad_at
            else:
                r = ctx.finish(res)
                assert r.bad_bits == 0
                assert_streams(snap_np(snap), wants[i], what="(batch %d)" % i)
    finally:
        q.close()
        for db in dbs:
            db.close()


def test_queue_empty_labels_need_the_exact_redo(ctx):
    """A batch whose domains have empty labels needs the exact-offset redo in regk_finish, which the single-buffered
    device outputs only allow with nothing queued behind it: REGK_ERR_STATE.  The batches after it still finish, and
    the same batch run alone equals the oracle."""
    batches = queue_batches()[:5]
    batches[1] = _records_case("empty_labels")
    ctx.set_types(batches[0].types)
    wants = [oracle.register_batch(b) for b in batches]
    dbs = [DeviceBatch(ctx, b, FLAG_OUT_DEVICE) for b in batches]
    q = Queue(ctx)
    try:
        _prime(ctx, q, dbs, wants)
        q.start()
        subs = [q.submit(db, None if i == 1 else q.reserve(w)) for i, (db, w) in enumerate(zip(dbs, wants))]
        for i, (res, snap) in enumerate(subs):
            if i == 1:
                with pytest.raises(RegkError) as ei:
                    ctx.finish(res)
                assert ei.value.code == REGK_ERR_STATE and "exact-offset redo" in ei.value.message
            else:
                assert ctx.finish(res).bad_bits == 0
                assert_streams(snap_np(snap), wants[i], what="(batch %d)" % i)
        q.close()
        res = ctx.register_raw(dbs[1].cb)
        assert res.launches >= 4                        # compose, then the exact redo's length and compose kernels
        assert_streams(fetch(res, batches[1].n), wants[1], what="(alone)")
    finally:
        q.close()
        for db in dbs:
            db.close()
