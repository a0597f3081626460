"""CPU tests of skip mode (REGK_SKIP_BAD): the per-record fence predicate and the ABI of regk_skipped.

fence_record() in regk_core.cuh is what the skip-mode fence pass runs on the GPU; here the same code, compiled with
g++ (tests/emul/skip_emul.cpp), is compared with the oracle's restatement of the fence (skip_util.fence_bits) record by
record, for every batch mode whose flags change what is fenced.
"""
import ctypes as C
import os
import random
import subprocess
import tempfile

import numpy as np
import pytest

from registrar_b200 import synth
from registrar_b200._native import host_cbatch
from registrar_b200.batch import FLAG_NO_JSON, FLAG_NO_PATH, FLAG_SKIP_BAD, RecordBatch
from skip_util import fence_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODES = {"host": 0, "alias": 0, "no_json": FLAG_NO_JSON, "no_path": FLAG_NO_PATH}


@pytest.fixture(scope="module")
def emul(built):
    """tests/emul/skip_emul.cpp built with g++ (seconds), again whenever the code it compiles has changed."""
    so = os.path.join(ROOT, "tests", "emul", "libskipemul.so")
    srcs = [os.path.join(ROOT, "tests", "emul", "skip_emul.cpp"),
            os.path.join(ROOT, "registrar_b200", "csrc", "regk_core.cuh"), os.path.join(ROOT, "include", "regk.h")]
    if not os.path.exists(so) or any(os.path.getmtime(so) < os.path.getmtime(f) for f in srcs):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unknown-pragmas",
                               "-fsanitize=undefined", "-fno-sanitize-recover=undefined", "-o", so, srcs[0]])
    lib = C.CDLL(so)
    lib.emul_fence.restype = C.c_uint32
    return lib


def emul_fence(emul, batch, flags):
    cb, keep = host_cbatch(batch, flags)
    bits = np.zeros(max(batch.n, 1), np.uint8)
    orr = emul.emul_fence(C.byref(cb), len(batch.types), bits.ctypes.data_as(C.c_void_p))
    del keep
    bits = bits[:batch.n]
    assert orr == int(np.bitwise_or.reduce(bits)) if batch.n else orr == 0
    return bits


def check_modes(emul, records, types, mutate_type=()):
    for mode, flags in MODES.items():
        alias = mode == "alias"
        batch = RecordBatch.from_records(records, types=types, alias=alias)
        for i in mutate_type:
            batch.type_id[i] = len(types) + (i % 3)         # outside the type table
        want = fence_bits(batch, flags)
        got = emul_fence(emul, batch, flags)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, (mode, int(bad[0]), batch.record(int(bad[0])), int(got[bad[0]]), int(want[bad[0]]))
        yield mode, want


def test_fence_matches_the_oracle_on_the_edge_rows(emul):
    from golden_util import as_record, load
    recs = [as_record(r["in"]) for r in load("edge.jsonl")]
    types = sorted({r["type"] for r in recs})
    seen = {}
    for mode, want in check_modes(emul, recs, types):
        seen[mode] = int(np.count_nonzero(want))
    assert seen["host"] > 5                                 # the fixture does exercise the fence


SPECIAL = [0x00, 0x2F, 0x22, 0x5C, 0x80, 0xFF, 0xC3, 0x7F, 0x1F, 0x20, 0x2E, 0x61, 0x41]


def _mutations(n_records, seed):
    base = synth.generate("config3", n=64, seed=seed)
    rng = random.Random(seed)
    recs, type_bad = [], []
    for i in range(n_records):
        r = base.record(rng.randrange(base.n))
        r = dict(r)
        field = rng.choice(["domain", "hostname", "address", "type", "empty", "dots"])
        if field in ("domain", "hostname", "address"):
            v = bytearray(r[field])
            pos = rng.randrange(len(v) + 1)
            c = rng.choice(SPECIAL) if rng.random() < 0.8 else rng.randrange(256)
            if pos < len(v) and rng.random() < 0.5:
                v[pos] = c                                  # replace a byte
            else:
                v.insert(pos, c)                            # insert one
            r[field] = bytes(v)
        elif field == "empty":
            r[rng.choice(["domain", "hostname", "address"])] = b""
        elif field == "dots":
            r["hostname"] = rng.choice([b".", b"..", b"...", b"./", b".a"])
        else:
            type_bad.append(i)
        recs.append(r)
    return recs, list(base.types), type_bad


@pytest.mark.parametrize("seed", [1, 2])
def test_fence_matches_the_oracle_on_single_byte_mutations(emul, seed):
    recs, types, type_bad = _mutations(3000, seed)          # 2 x 3000 mutated records, each checked in 4 modes
    counts = {}
    for mode, want in check_modes(emul, recs, types, type_bad):
        counts[mode] = {b: int(np.count_nonzero(want & b)) for b in (1, 2, 4, 8)}
    assert all(counts["host"][b] > 50 for b in (1, 2, 4, 8)), counts["host"]
    assert counts["alias"][2] == 0 and counts["no_json"][4] == counts["no_json"][8] == 0
    assert counts["no_path"][1] == counts["no_path"][2] == 0


def test_take_builds_the_batch_of_the_given_records():
    batch = synth.generate("config3", n=300)
    idx = [299, 0, 128, 127, 5, 5]
    sub = batch.take(idx)
    assert sub.n == len(idx)
    for k, i in enumerate(idx):
        assert sub.record(k) == batch.record(i)
    empty = batch.take([])
    assert empty.n == 0 and int(empty.domain_off[-1]) == 0
    var = RecordBatch.from_records([{"domain": "a.b", "hostname": "h%d" % (i * 7), "type": "host", "address": "1.2.3.%d" % i,
                                     "ports": list(range(i % 3))} for i in range(20)])
    assert var.host_off is not None
    sub = var.take([19, 3])
    assert sub.record(0) == var.record(19) and sub.record(1) == var.record(3)
    with pytest.raises(IndexError):
        batch.take([300])


def test_skipped_struct_layout_matches_header(built):
    from registrar_b200 import _native
    src = r"""
    #include <stddef.h>
    #include <stdio.h>
    #include "regk.h"
    int main(void) {
        printf("%zu %zu %zu %zu %zu %zu %u\n", sizeof(regk_skipped), offsetof(regk_skipped, n_skipped),
               offsetof(regk_skipped, flags), offsetof(regk_skipped, bad_bits), offsetof(regk_skipped, index),
               offsetof(regk_skipped, bits), (unsigned)REGK_SKIP_BAD);
        return 0;
    }
    """
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    S = _native.CSkipped
    assert got == [C.sizeof(S), S.n_skipped.offset, S.flags.offset, S.bad_bits.offset, S.index.offset, S.bits.offset,
                   FLAG_SKIP_BAD]
    assert "regk_skipped_records" in _native.EXPORTS
