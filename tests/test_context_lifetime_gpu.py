"""A context owns its CUDA resources and releases them on close: three contexts in a row in one process each run every
entry-point family and are closed, and the third computes what the first did; a context closed with an asynchronous
batch still in flight on a caller's torch stream leaves that stream usable; two live contexts on one device take turns
with growing shared-memory budgets (the limit a kernel may use is per device and kernel, shared by both)."""
import numpy as np
import pytest

from oracle import oracle
from registrar_b200 import synth
from registrar_b200.batch import RecordBatch, ServiceBatch, Snapshot

pytestmark = pytest.mark.gpu

ZK_CREATE, ZK_DELETE, ZK_GETDATA, ZK_SETDATA, ZK_REPLACE = 1, 2, 4, 5, 256


def _streams(r):
    return [np.asarray(a).tobytes() for a in (r.path_bytes, r.path_off, r.json_bytes, r.json_off)]


def _device_streams(res, n):
    import torch
    from registrar_b200 import multigpu
    dev = torch.device("cuda", 0)
    get = lambda p, c, dt: multigpu.device_tensor(p, c, dt, dev).cpu().numpy().tobytes()
    return [get(res.path_bytes, int(res.path_total), torch.uint8), get(res.path_off, n + 1, torch.int64),
            get(res.json_bytes, int(res.json_total), torch.uint8), get(res.json_off, n + 1, torch.int64)]


def _with_bad_record(hb, at):
    recs = [hb.record(i) for i in range(hb.n)]
    recs[at]["domain"] = recs[at]["domain"] + b"/x"
    return RecordBatch.from_records(recs, types=hb.types)


def every_family(ctx, n=3000):
    """Every entry-point family once on `ctx`; returns their host outputs, in order, as bytes."""
    import torch
    import replies_util as ru
    from registrar_b200 import multigpu
    from test_reconcile import _streams as record_streams, drift
    from test_read_replies import SESSION, model_of

    out = []
    hb, other = synth.generate("config3", n=n, seed=11), synth.generate("config1", n=n // 2, seed=12)
    want, want_other = _streams(oracle.register_batch(hb)), _streams(oracle.register_batch(other))
    # register: host and synchronous, the two async host sets, device-resident, pipelined, skip mode
    assert _streams(ctx.register_batch(hb)) == want
    ctx.set_option("async", 1)
    t1, t2 = ctx.submit(hb), ctx.submit(other)
    assert _streams(ctx.collect(t1, copy=True)) == want
    assert _streams(ctx.collect(t2, copy=True)) == want_other
    ctx.set_option("async", 0)
    cb, keep = multigpu.device_batch(hb, torch.device("cuda", 0))
    assert _device_streams(ctx.register_raw(cb), n) == want
    del keep
    ctx.set_option("chunk_records", 1024)
    assert _streams(ctx.register_batch(hb)) == want
    ctx.set_option("chunk_records", 262144)
    bad = _with_bad_record(hb, n // 3)
    skipped = ctx.register_batch(bad, skip_bad=True)
    assert skipped.skipped.tolist() == [n // 3]
    out += _streams(skipped) + [skipped.skipped_bits.tobytes()]
    # the calls on the batch finished last
    got = ctx.register_batch(hb)
    paths, pays = record_streams(got)
    parent_len, unique_first, _ = ctx.parent_dirs()
    out += [parent_len.tobytes(), unique_first.tobytes()]
    dirs = ctx.mkdirp_dirs()
    out += [dirs.dir_bytes.tobytes(), dirs.dir_off.tobytes(), dirs.depth_off.tobytes()]
    out += [ctx.mkdirp_requests(xid_base=5)[0].tobytes()]
    rec, dom, ports, _ = ctx.decode(last=True)
    out += [rec.tobytes(), dom.tobytes(), ports.tobytes()]
    # getData frames and their replies, then both reconcile calls and their repair frames
    fb, fo, _ = ctx.jute_requests(ZK_GETDATA, xid_base=3)
    out += [fb.tobytes(), fo.tobytes()]
    zk = model_of(paths, pays, skip=set(range(0, n, 9)))
    rep = ctx.read_replies(np.frombuffer(ru.replies(zk, fb), np.uint8))
    out += [rep.err.tobytes(), rep.node_rec.tobytes()]
    d = ctx.reconcile(Snapshot.from_nodes(drift(paths, pays, seed=3)))
    out += [d.cls.tobytes(), d.match.tobytes(), d.create.tobytes(), d.update.tobytes()]
    out += [ctx.reconcile_requests(op, xid_base=9)[0].tobytes() for op in (ZK_CREATE, ZK_SETDATA, ZK_DELETE)]
    d = ctx.reconcile_owned(rep, session=SESSION, zk_flags=1)
    assert rep.n_missing == d.n_create > 0
    out += [d.cls.tobytes(), d.create.tobytes()]
    out += [ctx.reconcile_requests(op, xid_base=9, observed_version=op != ZK_CREATE)[0].tobytes()
            for op in (ZK_CREATE, ZK_SETDATA, ZK_REPLACE)]
    # service records last: they reuse the payload buffers of the batch finished last
    services = [{"type": "service", "service": {"srvce": "_s%d" % i, "proto": "_tcp", "port": 80 + i, "ttl": 60}}
                for i in range(n // 4)]
    sv = ctx.service_records(ServiceBatch.from_services(services))
    out += [sv.json_bytes.tobytes(), sv.json_off.tobytes()]
    return out


def test_contexts_in_a_row_run_every_family(built):
    from registrar_b200 import _native
    first = None
    for _ in range(3):
        ctx = _native.Context(0)
        try:
            got = every_family(ctx)
        finally:
            ctx.close()
        first = first or got
    assert got == first


def close_in_flight(n=20000):
    """A context closed while an async host batch and a device batch are still queued on a caller's torch stream."""
    import torch
    from registrar_b200 import _native, multigpu
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    hb = synth.generate("config3", n=n, seed=4)
    ctx = _native.Context(0)
    ctx.set_stream(stream.cuda_stream)
    ctx.set_option("async", 1)
    ticket = ctx.submit(hb)
    cb, keep = multigpu.device_batch(hb, dev)
    ctx.register_raw(cb)
    ctx.close()
    x = torch.arange(1 << 20, device=dev, dtype=torch.int64)
    with torch.cuda.stream(stream):
        y = x * 3 + 1
    stream.synchronize()
    assert torch.equal(y.cpu(), torch.arange(1 << 20, dtype=torch.int64) * 3 + 1)
    del ticket, keep


def test_close_with_a_batch_in_flight_on_a_caller_stream(built):
    close_in_flight()


def alternating_budgets(n=5000):
    """Two live contexts take turns, each with a larger dom_cap than the other's last batch, then both go back down."""
    from registrar_b200 import _native
    hb = synth.generate("config3", n=n, seed=6)
    want = _streams(oracle.register_batch(hb))
    a, b = _native.Context(0), _native.Context(0)
    try:
        for k, cap in enumerate((2048, 4096, 8192, 16384, 32768, 49152, 2048, 4096)):
            ctx = (a, b)[k % 2]
            ctx.set_option("dom_cap", cap)
            assert _streams(ctx.register_batch(hb)) == want, cap
        for ctx in (a, b):
            ctx.set_option("dom_cap", 0)
            assert _streams(ctx.register_batch(hb)) == want
    finally:
        a.close()
        b.close()


def test_two_contexts_with_growing_shared_memory_budgets(built):
    alternating_budgets()
