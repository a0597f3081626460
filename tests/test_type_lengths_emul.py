"""The payload composers at every escaped type-name length, on the CPU (tests/emul), against the oracle.

A record's two type fragments, f1 = {"type":"T","address":" (22 + q bytes) and f2 = ,"T":{"address":" (16 + q bytes)
for a type T that escapes to q bytes, are copied by different code in regk_core.cuh depending on their length: f1 by
ten unconditional words up to 37 bytes and by the exact word loop beyond, f2 by put_frag_mid from 16 to 33 bytes and
by the exact word loop beyond.  Each is copied from one of four pre-shifted variants, by the byte phase of the output.
Every q from 0 to 80 (and 120, 255, 256, 1000) is reached by plain names, by names that grow through escapes (\\u00XX is
six bytes for one) and by names of multi-byte UTF-8, each at all 16 pairs of (f1 phase, f2 phase).  The GPU tests
(test_type_table_gpu.py) run the same matrix through the kernels.
"""
import ctypes as C
import json

import numpy as np
import pytest

from oracle import oracle
from registrar_b200.batch import RecordBatch
from test_core_emul import _blob, check_equal, run_emul

Q_LENGTHS = list(range(0, 81)) + [120, 255, 256, 1000]
ADDR_LENS = (1, 2, 3, 4, 17, 18, 19, 20)
TTLS = (0, 7, 42, 999, 123456, -5, 2147483647, -2147483647)
FILLER = b"h"                       # type of the records that shift the next record's byte phase

# (raw bytes, escaped length): escaping bytes, 0x7f (copied as is), 2-, 3- and 4-byte UTF-8
_ESCAPES = [(b"\x00", 6), (b'"', 2), (b"\x1f", 6), (b"\\", 2), (b"\n", 2), (b"\x01", 6), (b"\x7f", 1), (b"\x08", 2),
            (b"\x0b", 6), (b"\t", 2), (b"\x1e", 6), (b"\r", 2), (b"\x0c", 2)]
_UTF8 = [(c.encode(), len(c.encode())) for c in ("\u00e9", "\u20ac", "\u2028", "\ufffd", "\U0001f600", "\u0080",
                                                 "\u07ff", "\uffff", "\U0010ffff", "\u2029")]


def _fill(pieces, q, pad):
    """A name of escaped length q: `pieces` in turn while they fit, then `pad` bytes."""
    out, n, i = [], 0, 0
    while pieces and n + min(p[1] for p in pieces) <= q and i < 10 * q:
        raw, e = pieces[i % len(pieces)]
        i += 1
        if n + e <= q:
            out.append(raw)
            n += e
    return b"".join(out) + pad * (q - n)


def names_for(q):
    """Distinct type names of escaped length q: plain, escaping, UTF-8, and all of them mixed."""
    mixed = [p for pair in zip(_UTF8, _ESCAPES) for p in pair]
    cands = [b"t" * q, _fill(_ESCAPES, q, b"e"), _fill(_UTF8, q, b"u"), _fill(mixed, q, b"m")]
    out = []
    for c in cands:
        if c not in out:
            out.append(c)
    return out


def escaped_len(name):
    return len(oracle.quote_json_string(name)) - 2


def _json_len(q, al, ttl):
    return 22 + q + 16 + q + 2 * al + 4 + (0 if ttl is None else 7 + len(str(ttl)))


# filler records (address length, ttl) by the residue mod 4 of their payload length (type FILLER, q = 1)
_FILLERS = {1: (2, 10), 2: (1, None), 3: (1, 10)}


def type_records(names, start=0):
    """Records that put every name's f1 at each byte phase and, from there, its f2 at each byte phase: for each
    target phase of the record start, every address length of ADDR_LENS without ttl and with a ttl of some digit
    count, each behind a filler record that shifts the start to the target phase."""
    recs, pos = [], start
    for name in names:
        q = escaped_len(name)
        for p1 in range(4):
            for j, al in enumerate(ADDR_LENS):
                for ttl in (None, TTLS[(p1 * len(ADDR_LENS) + j) % len(TTLS)]):
                    need = (p1 - pos) % 4
                    if need:
                        fal, fttl = _FILLERS[need]
                        recs.append({"domain": b"f.example", "hostname": b"h", "type": FILLER,
                                     "address": b"8" * fal, "ttl": fttl})
                        pos += _json_len(1, fal, fttl)
                    recs.append({"domain": b"a.b", "hostname": b"h%d" % (al % 10), "type": name,
                                 "address": (b"10.0.0.%d" % al + b"0123456789abcdef")[:al], "ttl": ttl})
                    pos += _json_len(q, al, ttl)
    return recs


def type_tables(names, emul):
    """The names split into type tables (each with FILLER) that fit the 16 KB fragment budget."""
    tables, cur = [], []
    for nm in names:
        trial = cur + [nm]
        if _try_blob(emul, trial + [FILLER]) == 0:
            cur = trial
        else:
            assert cur, "a single name %r does not fit" % nm[:20]
            tables.append(cur)
            cur = [nm]
    if cur:
        tables.append(cur)
    return [t + [FILLER] for t in tables]


def _try_blob(emul, types):
    arr = (C.c_char_p * max(len(types), 1))(*types)
    lens = (C.c_uint32 * max(len(types), 1))(*[len(t) for t in types])
    out = (C.c_uint8 * 20000)()
    blen, maxq = C.c_uint32(0), C.c_uint32(0)
    return emul.emul_build_blob(arr, lens, len(types), out, 20000, C.byref(blen), C.byref(maxq))


def type_batches(qs, emul, alias=False):
    """One RecordBatch per type table over the names of every q in `qs`."""
    names = [nm for q in qs for nm in names_for(q)]
    return [RecordBatch.from_records(type_records(t[:-1]), types=t, alias=alias) for t in type_tables(names, emul)]


def phase_pairs(batch, want):
    """{type name: set of (f1 phase, f2 phase)} from the oracle's payload offsets."""
    pairs = {}
    for i in range(batch.n):
        name = batch.types[int(batch.type_id[i])]
        if name == FILLER:
            continue
        o = int(want.json_off[i])
        q = escaped_len(name)
        ttl = int(batch.ttl[i])
        al = int(batch.addr_off[i + 1] - batch.addr_off[i])
        o2 = o + 22 + q + al + (1 if ttl == -2 ** 31 else 8 + len(str(ttl)))
        assert want.json(i)[o2 - o:o2 - o + 2] == b',"', "f2 is not where it should be"
        pairs.setdefault(name, set()).add((o % 4, o2 % 4))
    return pairs


def test_names_reach_every_q():
    for q in Q_LENGTHS:
        names = names_for(q)
        assert [escaped_len(nm) for nm in names] == [q] * len(names)
        if q >= 6:
            assert len(names) == 4, q                   # with and without escapes, with and without UTF-8
    every = [nm for q in Q_LENGTHS for nm in names_for(q)]
    for raw, _ in _ESCAPES + _UTF8:                    # each escape and each UTF-8 width is used
        assert any(raw in nm for nm in every), raw


@pytest.mark.parametrize("generic", [0, 1])
@pytest.mark.parametrize("q", Q_LENGTHS)
def test_every_type_length(emul, q, generic):
    for batch in type_batches([q], emul):
        want, got_p, got_j = run_emul(emul, batch, generic)
        check_equal(want, got_p, got_j)
        for name, pairs in phase_pairs(batch, want).items():
            assert len(pairs) == 16, (q, name[:16], sorted(pairs))


@pytest.mark.parametrize("generic", [0, 1])
def test_type_lengths_in_one_table(emul, generic):
    """Many lengths in one table: fragments of different strides side by side in the blob, records of neighbouring
    lengths in one tile (and so sharing the boundary words of the output image)."""
    for batch in type_batches(range(0, 41), emul, alias=True):
        rng = np.random.default_rng(len(batch.types))
        batch = batch.take(rng.permutation(batch.n))
        check_equal(*run_emul(emul, batch, generic))


def largest_fitting(emul, make, others=()):
    """The largest k for which the table [make(k)] + others fits the fragment budget."""
    lo, hi = 0, 5000
    while lo < hi:
        m = (lo + hi + 1) // 2
        if _try_blob(emul, [make(m)] + list(others)) == 0:
            lo = m
        else:
            hi = m - 1
    return lo


ONE_BYTE_NAMES = [bytes([c]) for c in range(0x20, 0x7f) if not chr(c).isdigit() and c not in b'"\\']


def most_one_byte_types(emul):
    k = 0
    while k < len(ONE_BYTE_NAMES) and _try_blob(emul, ONE_BYTE_NAMES[:k + 1]) == 0:
        k += 1
    assert k < len(ONE_BYTE_NAMES)
    return k


def test_table_limits(emul):
    """The largest tables build_type_blob accepts stay within 16 KB; one byte more is refused as too large (2)."""
    for make in (lambda k: b"t" * k, lambda k: b"\x01" * k, lambda k: "\u20ac".encode() * k):
        k = largest_fitting(emul, make)
        blob, blen = _blob(emul, [make(k)])
        assert 15000 < blen <= 16384 and _try_blob(emul, [make(k + 1)]) == 2
    assert 1900 < largest_fitting(emul, lambda k: b"t" * k) < 2100
    k = most_one_byte_types(emul)
    blob, blen = _blob(emul, ONE_BYTE_NAMES[:k])
    assert 70 < k and blen <= 16384 and _try_blob(emul, ONE_BYTE_NAMES[:k + 1]) == 2


def _quote_ref(name: bytes) -> bytes:
    """ECMA-262 QuoteJSONString by Python's json module: lowercase \\u00xx, 0x7f and non-ASCII as they are."""
    return json.dumps(name.decode("utf-8"), ensure_ascii=False).encode("utf-8")


def test_escaping_matches_json_dumps(emul):
    """The oracle's escaping and the fragment table's bytes, all four pre-shifted variants, against Python's json."""
    names = list(dict.fromkeys([nm for q in Q_LENGTHS for nm in names_for(q)] +
                               [bytes([c]) for c in range(0x80) if not chr(c).isdigit()]))
    for nm in names:
        assert oracle.quote_json_string(nm) == _quote_ref(nm), nm
    for table in type_tables([nm for nm in names if nm not in (b"h", b"type")], emul):
        blob, blen = _blob(emul, table)
        raw = bytes(blob[:blen])
        frags = np.frombuffer(raw[:8 * len(table)], np.uint16).reshape(-1, 4)
        for name, (f1o, f1l, f2o, f2l) in zip(table, frags.tolist()):
            qj = _quote_ref(name)
            for off, ln, want in ((f1o, f1l, b'{"type":' + qj + b',"address":"'),
                                  (f2o, f2l, b"," + qj + b':{"address":"')):
                assert ln == len(want)
                stride = 4 * ((ln + 6) // 4)
                for k in range(4):
                    v = raw[off + k * stride:off + (k + 1) * stride]
                    assert v == b"\0" * k + want + b"\0" * (stride - k - ln), (name, k)


# --- the UTF-8 fence of regk_set_types ------------------------------------------------------------------------------

NOT_UTF8 = [
    b"\xc0\xaf", b"\xc1\xbf", b"\xe0\x80\xaf", b"\xe0\x9f\xbf", b"\xf0\x80\x80\xaf", b"\xf0\x8f\xbf\xbf",   # overlong
    b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xed\xa0\xbd\xed\xb8\x80", b"x\xed\xb0\x80y",                     # surrogates
    b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf7\xbf\xbf\xbf", b"\xf8\x88\x80\x80\x80", b"\xfe", b"\xff",  # > U+10FFFF
    b"\xc3", b"\xe2\x82", b"\xf0\x9f\x98", b"host\xe2\x82", b"\xe2\x82host", b"\xf0\x9f\x98\x80\xf0",       # truncated
    b"\x80", b"host\xbf", b"\xc3\xa9\xa9", b"\xe2\x82\xac\x80",                                            # stray
]
UTF8_EDGES = [b"\xc2\x80", b"\xdf\xbf", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\xef\xbf\xbd",
              b"\xef\xbf\xbf", b"\xf0\x90\x80\x80", b"\xf4\x8f\xbf\xbf", b"\xe2\x80\xa8", b"caf\xc3\xa9_host"]


def test_type_names_must_be_utf8(emul):
    for bad in NOT_UTF8:
        with pytest.raises(UnicodeDecodeError):
            bad.decode("utf-8")
        for k in range(3):
            table = [b"host", b"moray_host"]
            table.insert(k, bad)
            assert _try_blob(emul, table) == 1, (bad, k)
    for good in UTF8_EDGES:
        good.decode("utf-8")
        assert _try_blob(emul, [b"host", good]) == 0, good


def test_utf8_fence_agrees_with_python(emul):
    """Every 1- and 2-byte name and random short ones from a high-byte alphabet: accepted exactly when Python's
    strict UTF-8 decoder accepts them (names that collide with fixed keys or are array indices aside)."""
    rng = np.random.default_rng(2028)
    cands = [bytes([a]) for a in range(256)] + [bytes([a, b]) for a in range(256) for b in range(256)]
    alphabet = np.array([0x61, 0x7f, 0x80, 0x8f, 0x90, 0x9f, 0xa0, 0xbf, 0xc0, 0xc1, 0xc2, 0xdf, 0xe0, 0xe1, 0xec,
                         0xed, 0xee, 0xef, 0xf0, 0xf1, 0xf3, 0xf4, 0xf5, 0xff], np.uint8)
    for _ in range(20000):
        cands.append(rng.choice(alphabet, int(rng.integers(1, 7))).tobytes())
    for nm in cands:
        if nm.isdigit():
            continue
        try:
            nm.decode("utf-8")
            ok = True
        except UnicodeDecodeError:
            ok = False
        assert (_try_blob(emul, [nm]) == 0) == ok, nm
