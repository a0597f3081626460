"""Skip mode (REGK_SKIP_BAD) on the GPU: out-of-domain records come back empty and listed, everything else exactly
as a plain batch of the kept records alone, on every route of regk_register_batch."""
import random

import numpy as np
import pytest

from oracle import oracle
from registrar_b200 import synth
from registrar_b200.batch import (BAD_TOO_LARGE, FLAG_JOB_STEP, FLAG_NO_JSON, FLAG_NO_PATH, FLAG_SKIP_BAD,
                                  RecordBatch)
from skip_util import fence_bits

pytestmark = pytest.mark.gpu

MODES = {"host": 0, "alias": 0, "no_json": FLAG_NO_JSON, "no_path": FLAG_NO_PATH}
KINDS = ("domain", "host", "addr", "type")


@pytest.fixture(scope="module")
def ctx(built):
    from registrar_b200 import _native
    c = _native.Context(0)
    yield c
    c.close()


def corrupt(records, positions, kind, rng):
    """records[i] for i in positions made out of domain; returns the type-id positions to break after packing."""
    type_pos = []
    for i in positions:
        r = dict(records[i])
        if kind == "domain":
            d = bytearray(r["domain"])
            d.insert(rng.randrange(len(d) + 1), rng.choice([0x2F, 0x80, 0xE9]))
            r["domain"] = bytes(d)
        elif kind == "host":
            r["hostname"] = rng.choice([b"", b".", b"..", b"a/b", b"h\x00", b"\xffh"])
        elif kind == "addr":
            r["address"] = rng.choice([b"", b"1.2.3.\"4", b"\\", b"10.0.0.\x01", b"fe80::\xc3\xa9"])
        else:
            type_pos.append(i)
        records[i] = r
    return type_pos


def make(n, kind, positions, alias=False, seed=7, config="config3"):
    base = synth.generate(config, n=n, seed=seed)
    recs = [base.record(i) for i in range(n)]
    tpos = corrupt(recs, positions, kind, random.Random(seed))
    b = RecordBatch.from_records(recs, types=base.types, alias=alias)
    for i in tpos:
        b.type_id[i] = len(base.types)
    return b


def expected(batch, flags):
    bits = fence_bits(batch, flags)
    kept = np.nonzero(bits == 0)[0]
    ref = oracle.register_batch(batch.take(kept), flags_extra=flags)
    assert ref.bad_bits == 0
    before = np.zeros(batch.n + 1, np.int64)
    np.cumsum(bits == 0, out=before[1:])
    return bits, ref, before


def check(got, batch, flags):
    bits, ref, before = expected(batch, flags)
    bad = np.nonzero(bits)[0]
    assert np.array_equal(got.skipped, bad.astype(np.uint64))
    assert np.array_equal(got.skipped_bits, bits[bad])
    assert np.array_equal(np.asarray(got.path_off, np.uint64), ref.path_off[before]), "path offsets"
    assert np.array_equal(np.asarray(got.json_off, np.uint64), ref.json_off[before]), "payload offsets"
    assert np.array_equal(got.path_bytes, ref.path_bytes), "path bytes"
    assert np.array_equal(got.json_bytes, ref.json_bytes), "payload bytes"
    for i in bad[:50]:
        assert got.path(int(i)) == b"" and got.json(int(i)) == b""
    return bits


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("kind", KINDS)
def test_each_fault_kind_and_mode(ctx, kind, mode):
    n = 1000
    batch = make(n, kind, [0, 127, 128, 200, 201, n - 1], alias=mode == "alias")
    flags = MODES[mode]
    got = ctx.register_batch(batch, paths=not flags & FLAG_NO_PATH, payloads=not flags & FLAG_NO_JSON, skip_bad=True)
    bits = check(got, batch, flags)
    fenced = (kind == "domain" and mode != "no_path") or (kind == "host" and mode in ("host", "no_json")) or \
        (kind in ("addr", "type") and mode != "no_json")
    assert np.count_nonzero(bits) == (6 if fenced else 0)


def test_config3_with_one_percent_corrupted(ctx):
    n = 100_000
    rng = np.random.default_rng(3)
    pos = np.sort(rng.choice(n, n // 100, replace=False))
    base = synth.generate("config3", n=n)
    recs = [base.record(i) for i in range(n)]
    r = random.Random(3)
    tpos = []
    for k, kind in enumerate(KINDS):
        tpos += corrupt(recs, [int(i) for i in pos[k::4]], kind, r)
    batch = RecordBatch.from_records(recs, types=base.types)
    for i in tpos:
        batch.type_id[i] = 200
    got = ctx.register_batch(batch, skip_bad=True)
    assert got.skipped.size == pos.size
    check(got, batch, 0)


@pytest.mark.parametrize("bad", [False, True])
def test_single_record(ctx, bad):
    batch = make(1, "addr", [0] if bad else [])
    got = ctx.register_batch(batch, skip_bad=True)
    check(got, batch, 0)
    assert got.path_total == 0 if bad else got.path_total > 0


def test_all_records_bad(ctx):
    batch = make(300, "domain", range(300))
    got = ctx.register_batch(batch, skip_bad=True)
    check(got, batch, 0)
    assert got.skipped.size == 300 and got.path_total == 0 and got.json_total == 0
    assert not np.any(got.path_off) and not np.any(got.json_off)


def test_pipelined_host_route(ctx):
    ctx.set_option("chunk_records", 1024)
    try:
        n = 10_000
        batch = make(n, "host", [5, 1023, 1024, 4096, n - 1])
        got = ctx.register_batch(batch, skip_bad=True)
        check(got, batch, 0)
        clean = make(n, "host", [])
        assert np.array_equal(ctx.register_batch(clean, skip_bad=True).json_bytes, oracle.register_batch(clean).json_bytes)
    finally:
        ctx.set_option("chunk_records", 262144)


def test_async_dirty_and_clean_in_flight(ctx):
    dirty = make(5000, "type", [1, 2, 3, 4000])
    clean = synth.generate("config3", n=3000, seed=11)
    ctx.set_option("async", 1)
    try:
        t1 = ctx.submit(dirty, skip_bad=True)
        t2 = ctx.submit(clean, skip_bad=True)
        g1 = ctx.collect(t1, copy=True)
        g2 = ctx.collect(t2, copy=True)
    finally:
        ctx.set_option("async", 0)
    check(g1, dirty, 0)
    check(g2, clean, 0)
    assert g2.launches == 2


def test_device_resident_batch(ctx):
    import torch
    from registrar_b200 import _native, multigpu
    batch = make(2000, "domain", [0, 128, 1999])
    ctx.set_types(batch.types)
    cb, keep = multigpu.device_batch(batch, torch.device("cuda", 0))
    res = ctx.register_raw(cb, skip_bad=True)
    n = batch.n
    dev = torch.device("cuda", 0)
    got = _native.HostResult(
        n, multigpu.device_tensor(res.path_bytes, int(res.path_total), torch.uint8, dev).cpu().numpy(),
        multigpu.device_tensor(res.path_off, n + 1, torch.int64, dev).cpu().numpy().astype(np.uint64),
        multigpu.device_tensor(res.json_bytes, int(res.json_total), torch.uint8, dev).cpu().numpy(),
        multigpu.device_tensor(res.json_off, n + 1, torch.int64, dev).cpu().numpy().astype(np.uint64), 0, 0, 0, 0)
    got.skipped, got.skipped_bits = ctx.skipped_records()
    check(got, batch, 0)
    del keep


def test_offsets32(ctx):
    ctx.set_option("offsets32", 1)
    try:
        batch = make(3000, "addr", [7, 2999])
        got = ctx.register_batch(batch, skip_bad=True)
        assert got.path_off.dtype == np.uint32
        check(got, batch, 0)
    finally:
        ctx.set_option("offsets32", 0)


def test_force_generic(ctx):
    ctx.set_option("force_generic", 1)
    try:
        batch = make(1000, "host", [3, 500])
        got = ctx.register_batch(batch, skip_bad=True)
        check(got, batch, 0)
        assert got.generic_tiles > 0
    finally:
        ctx.set_option("force_generic", 0)


@pytest.mark.parametrize("mode", ["host", "alias"])
def test_dirty_batch_with_empty_labels(ctx, mode):
    batch = make(1000, "addr", [2, 129, 999], alias=mode == "alias")
    recs = [batch.record(i) for i in range(batch.n)]
    for i in (0, 130, 640):
        recs[i]["domain"] = b"a..b." + recs[i]["domain"]
    b2 = RecordBatch.from_records(recs, types=batch.types, alias=mode == "alias")
    got = ctx.register_batch(b2, skip_bad=True)
    check(got, b2, 0)


def test_clean_batch_is_untouched(ctx):
    batch = synth.generate("config3", n=50_000, seed=5)
    plain = ctx.register_batch(batch)
    skip = ctx.register_batch(batch, skip_bad=True)
    assert skip.launches == plain.launches == 2
    assert skip.skipped.size == 0 and skip.generic_tiles == 0
    for a in ("path_bytes", "path_off", "json_bytes", "json_off"):
        assert np.array_equal(getattr(skip, a), getattr(plain, a)), a


def test_refusals_still_hold(ctx):
    from registrar_b200._native import CResult, OutOfDomainError, RegkError, host_cbatch
    batch = make(500, "addr", [3])
    batch.addr_off = batch.addr_off.copy()
    batch.addr_off[10] = batch.addr_off[11] + 5              # corrupt offsets: REGK_BAD_TOO_LARGE
    with pytest.raises(OutOfDomainError) as e:
        ctx.register_batch(batch, skip_bad=True)
    assert e.value.result.bad_bits & BAD_TOO_LARGE
    with pytest.raises(RegkError) as e:
        ctx.skipped_records()
    assert e.value.code == 5                                  # REGK_ERR_STATE: the last batch was refused
    cb, keep = host_cbatch(make(10, "addr", []), FLAG_JOB_STEP | FLAG_SKIP_BAD)
    with pytest.raises(RegkError) as e:
        ctx.register_raw(cb, CResult())
    assert e.value.code == 1                                  # REGK_ERR_INVALID_ARG, before "no bound job"
    ctx.register_batch(make(10, "addr", []))
    with pytest.raises(RegkError) as e:
        ctx.skipped_records()                                 # plain batch finished last
    assert e.value.code == 5


def test_downstream_calls_see_the_kept_records(ctx):
    from registrar_b200._native import ZK_CREATE, ZK_DELETE
    batch = make(3000, "domain", [0, 127, 128, 1500, 2999])
    kept = batch.take(np.nonzero(fence_bits(batch, 0) == 0)[0])

    def downstream():
        out = [ctx.parent_dirs()[:2]]
        for op in (ZK_CREATE, ZK_DELETE):
            for group in (0, 7):
                out.append(ctx.jute_requests(op=op, group=group)[:2])
        rec, dom, ports, _ = ctx.decode(last=True)
        out.append((rec, dom, ports))
        return out
    ctx.register_batch(batch, skip_bad=True)
    a = downstream()
    ctx.register_batch(kept)
    b = downstream()
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert np.array_equal(u, v)


def test_no_lasting_effect_on_the_payload_budget(ctx):
    clean = synth.generate("config3", n=200_000, seed=9)
    ctx.register_batch(clean)
    dirty = make(200_000, "addr", list(range(0, 200_000, 97)))
    check(ctx.register_batch(dirty, skip_bad=True), dirty, 0)
    again = ctx.register_batch(clean)
    assert again.generic_tiles == 0
