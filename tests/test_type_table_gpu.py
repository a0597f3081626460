"""The type table on the GPU: the type-length matrix of test_type_lengths_emul.py through regk_register_batch on the
host and the device route, and the table itself at its limits - the largest table regk_set_types accepts and the first
it refuses, the most types, a type long enough to send its tiles down the global-memory route, the learned payload
budget meeting a longer type than it learned from, and the UTF-8 fence."""
import numpy as np
import pytest

import test_device_route_gpu as dr
import test_type_lengths_emul as tl
from oracle import oracle
from registrar_b200._native import REGK_ERR_INVALID_ARG, REGK_ERR_OUT_OF_DOMAIN, OutOfDomainError, RegkError
from registrar_b200.batch import BAD_TYPE_ID, RecordBatch

pytestmark = pytest.mark.gpu

TILE = 128


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def _fresh_context():
    from registrar_b200 import _native
    return _native.Context(0)


@pytest.mark.parametrize("route", ["host", "device"])
def test_type_matrix(ctx, emul, route):
    """Every escaped type length at every (f1, f2) byte phase pair: shared-memory tiles, force_generic, the unfused
    length kernel (no paths), and alias nodes."""
    dev = route == "device"
    for batch in tl.type_batches(tl.Q_LENGTHS, emul):
        dr.check_route(ctx, batch, dev, dev, modes=("default", "force_generic", "no_path"))
    for batch in tl.type_batches(tl.Q_LENGTHS, emul, alias=True):
        dr.check_route(ctx, batch, dev, dev, modes=("default", "force_generic"))


def _records(types, type_ids, ttl=5, addr=b"10.1.2.3"):
    return RecordBatch.from_records([{"domain": b"svc.dc.example.com", "hostname": b"h%05d" % i, "type": types[t],
                                      "address": addr, "ttl": ttl} for i, t in enumerate(type_ids)], types=types)


def _same(got, want):
    assert want.bad_bits == 0
    assert np.array_equal(got.path_off, want.path_off) and np.array_equal(got.path_bytes, want.path_bytes)
    assert np.array_equal(got.json_off, want.json_off) and np.array_equal(got.json_bytes, want.json_bytes)


def test_largest_table_and_the_first_refused(ctx, emul):
    for make in (lambda k: b"t" * k, lambda k: b"\x01" * k):
        k = tl.largest_fitting(emul, make)
        table = [make(k)]
        batch = _records(table, [0] * 300)
        for route in (False, True):
            dr.check_route(ctx, batch, route, route, modes=("default",))
        with pytest.raises(RegkError) as ei:
            ctx.set_types([make(k + 1)])
        assert ei.value.code == REGK_ERR_INVALID_ARG
        _same(ctx.register_batch(batch), oracle.register_batch(batch))    # the refused call left the table in force


def test_most_types(ctx, emul):
    k = tl.most_one_byte_types(emul)
    table = tl.ONE_BYTE_NAMES[:k]
    ids = [i % k for i in range(3 * k + 50)]
    batch = _records(table, ids)
    assert set(batch.type_id.tolist()) == set(range(k))
    for route in (False, True):
        dr.check_route(ctx, batch, route, route, modes=("default", "force_generic"))
    bad_at = k + 5
    batch.type_id[bad_at] = k                                            # one past the last type
    want = oracle.register_batch(batch)
    assert want.bad_bits == BAD_TYPE_ID and want.first_bad == bad_at
    with pytest.raises(OutOfDomainError) as ei:
        ctx.register_batch(batch)
    assert ei.value.result.bad_bits == BAD_TYPE_ID and ei.value.result.first_bad == bad_at
    with pytest.raises(RegkError) as ei:
        ctx.set_types(tl.ONE_BYTE_NAMES[:k + 1])
    assert ei.value.code == REGK_ERR_INVALID_ARG


def test_long_type_goes_generic_tile_by_tile(ctx, emul):
    """A type of about 2000 escaped bytes next to short ones: a tile of 128 such records (over 500 KB of payload) takes
    the global-memory route, a tile with one of them among short records composes in shared memory."""
    short = [b"host", b"db_host"]
    q = tl.largest_fitting(emul, lambda k: b"t" * k, short)
    assert q > 1900
    table = short + [b"t" * q]
    ntiles = 8
    ids = [i % 2 for i in range(ntiles * TILE)]
    long_tiles = (1, 5)
    for t in long_tiles:
        ids[t * TILE:(t + 1) * TILE] = [2] * TILE
    ids[3 * TILE + 77] = 2
    batch = _records(table, ids)
    want = oracle.register_batch(batch)
    tile_bytes = np.diff(want.json_off[::TILE].astype(np.int64).tolist() + [int(want.json_off[-1])])
    assert all(tile_bytes[t] > 98304 for t in long_tiles) and tile_bytes[3] < 32768
    for route in (False, True):
        res, got = dr.run_route(ctx, batch, route, route)
        dr.assert_streams(got, want)
        assert res.generic_tiles == len(long_tiles), route
        dr.check_route(ctx, batch, route, route, want=want, modes=("force_generic", "no_path"))


def test_learned_payload_budget_meets_a_longer_type(emul):
    """The payload kernel sizes its shared-memory image from the bytes per record of the batch finished last (same
    a-priori estimate).  A batch of the same address and port bytes but a longer type overflows that budget: its tiles
    go generic (still exact), learning is switched off, and the same batch again fits the a-priori budget.  A new
    type table starts the learning again."""
    ctx = _fresh_context()
    try:
        n = 8192
        long_q = 60
        table = [b"host", b"l" * long_q]
        a, b = _records(table, [0] * n, ttl=5), _records(table, [1] * n, ttl=5)
        assert a.addr_bytes.size == b.addr_bytes.size
        want_a, want_b = oracle.register_batch(a), oracle.register_batch(b)
        # the a-priori estimate (the longest type counted twice) covers b's records
        est = 42 + 2 * long_q + 2 * len(b"10.1.2.3") + 11 + 2
        assert int(want_b.json_off[-1]) // n <= est
        ra = ctx.register_batch(a)
        _same(ra, want_a)
        assert ra.generic_tiles == 0
        rb = ctx.register_batch(b)
        _same(rb, want_b)
        assert rb.generic_tiles > 0                     # the budget learned from a was too small
        rc = ctx.register_batch(b)
        _same(rc, want_b)
        assert rc.generic_tiles == 0                    # learning is off: the a-priori budget
        ctx.set_types(table + [b"x"])                   # a new table: learning starts again
        a2 = _records(table + [b"x"], [0] * n, ttl=5)
        b2 = _records(table + [b"x"], [1] * n, ttl=5)
        assert ctx.register_batch(a2).generic_tiles == 0
        rb2 = ctx.register_batch(b2)
        _same(rb2, oracle.register_batch(b2))
        assert rb2.generic_tiles > 0
    finally:
        ctx.close()


def test_type_names_must_be_utf8(ctx):
    good = [b"host", b"moray_host"]
    batch = _records(good, [0, 1] * 100)
    ctx.set_types(good)
    for bad in tl.NOT_UTF8:
        with pytest.raises(OutOfDomainError) as ei:
            ctx.set_types([b"host", bad, b"moray_host"])
        assert ei.value.code == REGK_ERR_OUT_OF_DOMAIN and "type 1 " in ei.value.message, bad
    _same(ctx.register_batch(batch), oracle.register_batch(batch))
    edges = tl.UTF8_EDGES
    batch = _records(edges, list(range(len(edges))) * 20)
    _same(ctx.register_batch(batch), oracle.register_batch(batch))
