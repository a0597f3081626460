"""An independent restatement of REGK_RESOLVE_ANY_FORM (include/regk.h), written from the reference README's prose
(README.md:441-755, "About TTLs" :670-755) on top of resolve_util.

The canonical reader decides first (resolve_util.record).  A node it refuses, with data and a path, is read by the
general rules: json.loads on the latin-1 decoded bytes (strict, NaN and Infinity refused), member pairs kept in order
so the last of a name wins, every string taken as its raw token (escapes left as they are), every number as its raw
text; nesting depth and escaped member names are checked on the parsed tree.  The records it yields have
resolve_util.record's shape, so class, answers and text follow resolve_util's rules unchanged."""
import json
import re

import resolve_util as rv

MAX_DEPTH = 64
U32 = (0, 2 ** 32 - 1)
_STR = re.compile(r'"((?:[^"\\]|\\.)*)"', re.S)


class _Obj(list):
    pass


class _Num:
    def __init__(self, text, integral):
        self.text, self.integral = text, integral


class _Other:
    pass


_ABSENT = object()


def _refuse(name):
    raise ValueError("not a JSON number: " + name)


def parse(data: bytes):
    """the raw tree (_Obj of (raw name, value) pairs, lists, raw string bytes, _Num, _Other), or None when data is not
    one JSON object within the depth limit with unescaped member names"""
    s = data.decode("latin-1")
    try:
        tree = json.loads(s, strict=True, object_pairs_hook=_Obj, parse_int=lambda t: _Num(t, True),
                          parse_float=lambda t: _Num(t, False), parse_constant=_refuse)
    except (ValueError, RecursionError):
        return None
    toks = iter(_STR.findall(s))
    bad = []

    def walk(v, depth):
        if isinstance(v, (_Obj, list)) and depth + 1 > MAX_DEPTH:
            bad.append("depth")
        if isinstance(v, _Obj):
            out = _Obj()
            for _, x in v:
                k = next(toks).encode("latin-1")
                if b"\\" in k:
                    bad.append("escaped name")
                out.append((k, walk(x, depth + 1)))
            return out
        if isinstance(v, list):
            return [walk(x, depth + 1) for x in v]
        if isinstance(v, str):
            return next(toks).encode("latin-1")
        if isinstance(v, _Num):
            return v
        return _Other()
    raw = walk(tree, 0)
    return raw if isinstance(raw, _Obj) and not bad else None


def _get(obj, name):
    """the last member called name, or _ABSENT"""
    v = _ABSENT
    for k, x in obj:
        if k == name:
            v = x
    return v


def _int(v, lo, hi):
    """the value of an integer token in [lo, hi], else None"""
    if not isinstance(v, _Num) or not v.integral or v.text == "-0" or len(v.text) > 12:
        return None
    x = int(v.text)
    return x if lo <= x <= hi else None


def _ttls(*vals):
    """(ok, the first present ttl or None)"""
    got = []
    for v in vals:
        if v is _ABSENT:
            continue
        x = _int(v, *rv.I32)
        if x is None:
            return False, None
        got.append(x)
    return True, (got[0] if got else None)


def general(data: bytes):
    """the general reader's record, resolve_util.record's shape, or None"""
    t = parse(data)
    if t is None:
        return None
    typ = _get(t, b"type")
    if not isinstance(typ, bytes):
        return None
    if typ == b"service":
        mid = _get(t, b"service")
        if not isinstance(mid, _Obj):
            return None
        sin = _get(mid, b"service")
        if not isinstance(sin, _Obj):
            return None
        srvce, proto, port = _get(sin, b"srvce"), _get(sin, b"proto"), _int(_get(sin, b"port"), *U32)
        ok, ttl = _ttls(_get(sin, b"ttl"), _get(mid, b"ttl"), _get(t, b"ttl"))
        if not (isinstance(srvce, bytes) and isinstance(proto, bytes) and port is not None and ok):
            return None
        return ("service", srvce, proto, port, ttl)
    inner = _get(t, typ)
    if not isinstance(inner, _Obj):
        return None
    addr = _get(inner, b"address")
    if not isinstance(addr, bytes):
        return None
    ports = _get(inner, b"ports")
    if ports is _ABSENT:
        ports = None
    elif isinstance(ports, list) and all(_int(p, *U32) is not None for p in ports):
        ports = [_int(p, *U32) for p in ports]
    else:
        return None
    ok, ttl = _ttls(_get(inner, b"ttl"), _get(t, b"ttl"))
    if not ok:
        return None
    return ("host", typ, addr, ttl, ports)


def record(path: bytes, data: bytes, any_form: bool):
    """(canonical record or None, general record or None): the general one only for a candidate"""
    canon = rv.record(data) if path.startswith(b"/") else None
    cand = any_form and canon is None and bool(data) and path.startswith(b"/")
    return canon, (general(data) if cand else None)


def classify(path: bytes, data: bytes, any_form: bool):
    """(class, record): resolve_util.classify's rules on the record the two readers give"""
    canon, gen = record(path, data, any_form)
    if gen is None:
        return rv.classify(path, data)
    name = rv.name_of(path)
    names = [name] + ([gen[1] + b"." + gen[2] + b"." + name] if gen[0] == "service" else [])
    if not all(rv.valid_name(x) for x in names):
        return rv.BAD_NAME, gen
    if gen[0] == "host":
        if gen[1] not in rv.QUERYABLE | rv.USABLE:
            return rv.UNKNOWN_TYPE, gen
        if not rv.valid_ipv4(gen[2]):
            return rv.BAD_ADDRESS, gen
    ttl = gen[4] if gen[0] == "service" else gen[3]
    if ttl is not None and ttl < 0:
        return rv.BAD_TTL, gen
    ports = [gen[3]] if gen[0] == "service" else (gen[4] or [])
    if any(p > 65535 for p in ports):
        return rv.BAD_PORT, gen
    return rv.OK, gen


def canonical(rec):
    """the canonical payload of a record (its strings verbatim): what resolve_util.record reads back as rec"""
    if rec[0] == "service":
        _, srvce, proto, port, ttl = rec
        inner = b'{"srvce":"%s","proto":"%s","port":%d%s}' % (srvce, proto, port, b"" if ttl is None else b',"ttl":%d' % ttl)
        return b'{"type":"service","service":{"type":"service","service":%s}}' % inner
    _, typ, addr, ttl, ports = rec
    return b'{"type":"%s","address":"%s"%s,"%s":{"address":"%s"%s}}' % (
        typ, addr, b"" if ttl is None else b',"ttl":%d' % ttl, typ, addr,
        b"" if ports is None else b',"ports":[%s]' % b",".join(b"%d" % p for p in ports))


def restated(nodes, any_form: bool):
    """nodes with every payload the general reader reads (as a record that is not NOT_RECORD) replaced by its canonical
    form: resolve_util then gives exactly the flagged answers, so its resolve, dns_util and dns_ptr_util apply as they
    are.  A record whose strings hold bytes json.loads cannot read as UTF-8 is kept as it is."""
    out = []
    for path, data in nodes:
        _, gen = record(path, data, any_form)
        if gen is not None:
            c = canonical(gen)
            assert rv.record(c) == gen, (data, c)
            data = c
        out.append((path, data))
    return out


def resolve(nodes, dh, ds, any_form: bool):
    """resolve_util.resolve's result for the snapshot, with REGK_RESOLVE_ANY_FORM's records when any_form"""
    index, cls, recs = {}, [], []
    for j, (path, data) in enumerate(nodes):
        if path in index:
            raise rv.DuplicateNode(j)
        index[path] = j
    want = rv.resolve(restated(nodes, any_form), dh, ds)
    for j, (path, data) in enumerate(nodes):
        c, _ = classify(path, data, any_form)
        assert c == want["node_cls"][j], (path, data, c, want["node_cls"][j])
    return want
