"""The compose kernels' L2 lookahead on batches longer than a wave (each CTA prefetches the offset and metadata
slices of the tile half a wave ahead, 500-700 tiles on an H100, and the payload kernel also that tile's address bytes
and port values, between offsets it loads unvalidated): results equal the oracle on every route, and corrupt offsets
in tiles that other CTAs prefetch for are refused exactly as the composers' own checks refuse them."""
import numpy as np
import pytest

from oracle import oracle
from registrar_b200 import synth
from registrar_b200.batch import BAD_TOO_LARGE, RecordBatch

pytestmark = pytest.mark.gpu

TILE = 128


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def assert_same(got, want):
    assert want.bad_bits == 0
    assert np.array_equal(got.path_off, want.path_off), "path offsets"
    assert np.array_equal(got.json_off, want.json_off), "payload offsets"
    assert np.array_equal(got.path_bytes, want.path_bytes), "path bytes"
    assert np.array_equal(got.json_bytes, want.json_bytes), "payload bytes"


def wave_tiles(ctx):
    return 8 * ctx.get_option("sm_count")            # the path kernel's resident CTAs on the benchmark configs


@pytest.mark.parametrize("config,n", [("config3", 400_000), ("config5", 300_000), ("config2", 300_000)])
def test_longer_than_a_wave(ctx, config, n):
    assert n // TILE > 2 * wave_tiles(ctx)
    batch = synth.generate(config, n=n, start=12_345)
    got = ctx.register_batch(batch)
    assert_same(got, oracle.register_batch(batch))
    if config != "config5":
        assert got.generic_tiles == 0


def test_device_resident_batch(ctx):
    import torch
    from registrar_b200 import multigpu
    n = 500_000
    batch = synth.generate("config3", n=n, start=77)
    cb, keep = multigpu.device_batch(batch, torch.device("cuda", 0))
    r = ctx.register_raw(cb)
    dev = torch.device("cuda", 0)
    want = oracle.register_batch(batch)
    assert np.array_equal(multigpu.device_tensor(r.path_off, n + 1, torch.int64, dev).cpu().numpy().astype(np.uint64),
                          want.path_off)
    assert np.array_equal(multigpu.device_tensor(r.json_off, n + 1, torch.int64, dev).cpu().numpy().astype(np.uint64),
                          want.json_off)
    assert np.array_equal(multigpu.device_tensor(r.path_bytes, int(r.path_total), torch.uint8, dev).cpu().numpy(),
                          want.path_bytes)
    assert np.array_equal(multigpu.device_tensor(r.json_bytes, int(r.json_total), torch.uint8, dev).cpu().numpy(),
                          want.json_bytes)
    del keep


def test_variable_hostnames_and_alias(ctx):
    base = synth.generate("config3", n=300_000, start=5)
    recs = [base.record(i) for i in range(base.n)]
    for i, r in enumerate(recs):
        r["hostname"] = b"h%x" % (i * 2654435761 % (1 << (4 + i % 60)))
    for alias in (False, True):
        batch = RecordBatch.from_records(recs, types=base.types, alias=alias)
        assert alias or batch.host_off is not None
        assert_same(ctx.register_batch(batch), oracle.register_batch(batch))


def test_pipelined_host_route(ctx):
    # three chunks of 2 048 tiles: the lookahead stops half a wave before each chunk's end
    batch = synth.generate("config3", n=700_000, start=3)
    got = ctx.register_batch(batch)
    assert got.launches == 2 * 3
    assert_same(got, oracle.register_batch(batch))


def test_skip_mode_long_batch(ctx):
    base = synth.generate("config3", n=300_000, start=9)
    recs = [base.record(i) for i in range(base.n)]
    bad = [150_001, 299_990]
    for i in bad:
        recs[i] = dict(recs[i], domain=recs[i]["domain"] + b"/x")
    batch = RecordBatch.from_records(recs, types=base.types)
    got = ctx.register_batch(batch, skip_bad=True)
    assert np.array_equal(got.skipped, np.array(bad, np.uint64))
    keep = np.setdiff1d(np.arange(batch.n), bad)
    want = oracle.register_batch(batch.take(keep))
    assert np.array_equal(got.path_bytes, want.path_bytes) and np.array_equal(got.json_bytes, want.json_bytes)


def too_large_first(off, lo_limit_tiles, limit):
    """First record a compose kernel reports REGK_BAD_TOO_LARGE for, given one offsets array of the batch: a tile whose
    extents are reversed or past the buffer refuses all its records; otherwise a record whose own offsets are reversed
    or outside its tile's extents (path kernel, lo_limit_tiles) or past the buffer (payload kernel)."""
    off = off.astype(np.int64)
    n = len(off) - 1
    bad = np.zeros(n, bool)
    d0, d1 = off[:-1], off[1:]
    if lo_limit_tiles:
        for t0 in range(0, n, TILE):
            t1 = min(t0 + TILE, n)
            D0, D1 = off[t0], off[t1]
            if D1 < D0 or D1 > limit:
                bad[t0:t1] = True
            else:
                bad[t0:t1] |= ~((d1[t0:t1] >= d0[t0:t1]) & (d0[t0:t1] >= D0) & (d1[t0:t1] <= D1))
    else:
        bad = (d1 < d0) | (d1 > limit)
    return int(np.argmax(bad)) if bad.any() else None


@pytest.mark.parametrize("case", ["dom_decreasing", "dom_past_end", "dom_tile_boundary", "addr_decreasing",
                                  "addr_past_end", "addr_tile_boundary", "ports_past_end", "ports_tile_boundary"])
def test_corrupt_offsets_in_a_lookahead_tile(ctx, case):
    """Offsets in a tile that CTAs earlier in the grid prefetch for (the payload kernel sizes its address and port
    prefetches from addr_off / ports_off): the batch is refused with the same bits and first index as the composers'
    own checks give."""
    from registrar_b200._native import OutOfDomainError
    n = 300_000
    batch = synth.generate("config3", n=n, start=1)
    w = wave_tiles(ctx)
    i = (w + 37) * TILE + 45                       # past the first wave: some earlier CTA prefetches this tile
    field, path_side = {"dom": ("domain_off", True), "add": ("addr_off", False), "por": ("ports_off", False)}[case[:3]]
    arr = getattr(batch, field).copy()
    if case.endswith("tile_boundary"):                 # an entry the payload kernel's lookahead loads as a bound
        i = (w + 90) * TILE
    if case.endswith("decreasing"):
        arr[i] = arr[i - 2]
    else:
        arr[i] = 2 ** 31 - 16
    setattr(batch, field, arr)
    limit = {"domain_off": len(batch.domain_bytes), "addr_off": len(batch.addr_bytes),
             "ports_off": len(batch.ports)}[field]
    want_first = too_large_first(arr, path_side, limit)
    assert want_first is not None and want_first >= w * TILE
    with pytest.raises(OutOfDomainError) as ei:
        ctx.register_batch(batch)
    assert ei.value.result.bad_bits & BAD_TOO_LARGE
    assert ei.value.result.first_bad == want_first
