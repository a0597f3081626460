"""An independent restatement of regk_resolve, written from the reference README's prose (README.md:274-282 type tables,
:441-755 host and service records, SRV answers and TTLs): Python string operations on paths, json.loads on payloads.

A payload is a record when json.loads accepts it and it is in the compact canonical form this library writes: rebuilt
from the parsed structure with every string taken verbatim from the payload (escapes left as they are), it must equal
the payload byte for byte.  Payloads that are not JSON are not modelled beyond "not a record"."""
import json
import re

OK, EMPTY, NOT_RECORD, BAD_NAME, UNKNOWN_TYPE, BAD_ADDRESS, BAD_TTL, BAD_PORT = range(8)
HOST_A, SERVICE_A, SERVICE_SRV = 1, 2, 3
QUERYABLE = {b"db_host", b"host", b"load_balancer", b"moray_host", b"redis_host"}
USABLE = {b"load_balancer", b"moray_host", b"ops_host", b"redis_host", b"rr_host"}
I32 = (-2 ** 31, 2 ** 31 - 1)

_STR = re.compile(rb'"((?:[^"\\]|\\.)*)"', re.S)
_LABEL = re.compile(rb"[A-Za-z0-9_-]{1,63}")
_OCTET = re.compile(rb"0|[1-9][0-9]{0,2}")


class DuplicateNode(ValueError):
    def __init__(self, j):
        super().__init__("node %d repeats an earlier path" % j)
        self.node = j


class _Obj(list):
    pass


class _Bad:
    pass


def _raw(data: bytes):
    """(k, v) pairs with every string as its raw bytes, or None when data is not canonical compact JSON"""
    try:
        tree = json.loads(data, object_pairs_hook=_Obj)
    except ValueError:
        return None
    toks = iter(_STR.findall(data))

    def walk(v):
        if isinstance(v, _Obj):
            return _Obj((next(toks), walk(x)) for _, x in v)
        if isinstance(v, list):
            return [walk(x) for x in v]
        if isinstance(v, str):
            return next(toks)
        if isinstance(v, int) and not isinstance(v, bool):
            return v
        return _Bad()

    def ser(v):
        if isinstance(v, _Obj):
            return b"{" + b",".join(b'"' + k + b'":' + ser(x) for k, x in v) + b"}"
        if isinstance(v, list):
            return b"[" + b",".join(ser(x) for x in v) + b"]"
        if isinstance(v, bytes):
            return b'"' + v + b'"'
        if isinstance(v, int):
            return str(v).encode()
        return b"\0"
    raw = walk(tree)
    return raw if ser(raw) == data else None


def _int(v, lo, hi):
    return isinstance(v, int) and lo <= v <= hi


def record(data: bytes):
    """("service", srvce, proto, port, ttl|None) or ("host", type, address, ttl|None, ports|None), or None"""
    t = _raw(data)
    if not isinstance(t, _Obj) or not t or t[0][0] != b"type" or not isinstance(t[0][1], bytes):
        return None
    if t[0][1] == b"service" and len(t) == 2 and t[1][0] == b"service" and isinstance(t[1][1], _Obj):
        inner = t[1][1]
        if len(inner) == 2 and inner[0] == (b"type", b"service") and inner[1][0] == b"service" and isinstance(inner[1][1], _Obj):
            mem = inner[1][1]
            keys = [k for k, _ in mem]
            d = dict(mem)
            if (len(keys) == len(set(keys)) and set(keys) <= {b"srvce", b"proto", b"port", b"ttl"}
                    and {b"srvce", b"proto", b"port"} <= set(keys) and isinstance(d[b"srvce"], bytes)
                    and isinstance(d[b"proto"], bytes) and _int(d[b"port"], 0, 2 ** 32 - 1)
                    and (b"ttl" not in d or _int(d[b"ttl"], *I32))):
                return ("service", d[b"srvce"], d[b"proto"], d[b"port"], d.get(b"ttl"))
    typ = t[0][1]
    rest = list(t[1:])
    if not rest or rest[0][0] != b"address" or not isinstance(rest[0][1], bytes):
        return None
    addr = rest.pop(0)[1]
    ttl = None
    if rest and rest[0][0] == b"ttl":
        ttl = rest.pop(0)[1]
        if not _int(ttl, *I32):
            return None
    if len(rest) != 1 or rest[0][0] != typ or not isinstance(rest[0][1], _Obj):
        return None
    inner = list(rest[0][1])
    if not inner or inner[0] != (b"address", addr):
        return None
    ports = None
    if len(inner) == 2 and inner[1][0] == b"ports" and isinstance(inner[1][1], list):
        ports = inner[1][1]
        if not all(_int(p, 0, 2 ** 32 - 1) for p in ports):
            return None
    elif len(inner) != 1:
        return None
    return ("host", typ, addr, ttl, ports)


def name_of(path: bytes) -> bytes:
    """/us/joyent/example/b44c74d6 -> b44c74d6.example.joyent.us"""
    return b".".join(reversed(path[1:].split(b"/")))


def valid_name(name: bytes) -> bool:
    return len(name) <= 253 and all(_LABEL.fullmatch(label) for label in name.split(b"."))


def valid_ipv4(a: bytes) -> bool:
    parts = a.split(b".")
    return len(parts) == 4 and all(_OCTET.fullmatch(x) and int(x) <= 255 for x in parts)


def classify(path: bytes, data: bytes):
    """(class, record)"""
    if not data:
        return EMPTY, None
    rec = record(data) if path.startswith(b"/") else None
    if rec is None:
        return NOT_RECORD, None
    name = name_of(path)
    names = [name] + ([rec[1] + b"." + rec[2] + b"." + name] if rec[0] == "service" else [])
    if not all(valid_name(x) for x in names):
        return BAD_NAME, rec
    if rec[0] == "host":
        if rec[1] not in QUERYABLE | USABLE:
            return UNKNOWN_TYPE, rec
        if not valid_ipv4(rec[2]):
            return BAD_ADDRESS, rec
    ttl = rec[4] if rec[0] == "service" else rec[3]
    if ttl is not None and ttl < 0:
        return BAD_TTL, rec
    ports = [rec[3]] if rec[0] == "service" else (rec[4] or [])
    if any(p > 65535 for p in ports):
        return BAD_PORT, rec
    return OK, rec


def a_line(name, ttl, addr):
    return b"%s.\t%d\tIN\tA\t%s\n" % (name, ttl, addr)


def srv_line(srvce, proto, service, ttl, port, child):
    return b"%s.%s.%s.\t%d\tIN\tSRV\t0 10 %d %s.\n" % (srvce, proto, service, ttl, port, child)


def resolve(nodes, default_host_ttl, default_srv_ttl):
    """nodes = [(path, data)] -> {"q_kind", "q_node", "sections": [(answer, additional)], "node_cls", "unresolved",
    "n_answers", "n_additional"}"""
    index, cls, recs = {}, [], []
    for j, (path, data) in enumerate(nodes):
        if path in index:
            raise DuplicateNode(j)
        index[path] = j
        c, r = classify(path, data)
        cls.append(c)
        recs.append(r)

    def is_service(j):
        return cls[j] == OK and recs[j][0] == "service"

    def a_ttl(j):
        return default_host_ttl if recs[j][3] is None else recs[j][3]

    def srv_ttl(j):
        return default_srv_ttl if recs[j][4] is None else recs[j][4]

    children = {}
    for j, (path, _) in enumerate(nodes):
        if cls[j] != OK or recs[j][0] != "host" or recs[j][1] not in USABLE:
            continue
        k = index.get(path[:path.rfind(b"/")]) if path.rfind(b"/") > 0 else None
        if k is not None and is_service(k):
            children.setdefault(k, []).append(j)
    out = {"q_kind": [], "q_node": [], "sections": [], "node_cls": cls, "n_answers": 0, "n_additional": 0,
           "unresolved": [j for j, c in enumerate(cls) if c >= NOT_RECORD]}

    def add(kind, j, answer, additional, n_ans, n_add):
        out["q_kind"].append(kind)
        out["q_node"].append(j)
        out["sections"].append((answer, additional))
        out["n_answers"] += n_ans
        out["n_additional"] += n_add

    for j, (path, _) in enumerate(nodes):
        if cls[j] != OK:
            continue
        name = name_of(path)
        if recs[j][0] == "host" and recs[j][1] in QUERYABLE:
            add(HOST_A, j, a_line(name, a_ttl(j), recs[j][2]), b"", 1, 0)
        elif recs[j][0] == "service":
            _, srvce, proto, port, _ = recs[j]
            kids = children.get(j, [])
            a = b"".join(a_line(name, min(srv_ttl(j), a_ttl(c)), recs[c][2]) for c in kids)
            add(SERVICE_A, j, a, b"", len(kids), 0)
            srv, extra, n_srv, n_extra = b"", b"", 0, 0
            for c in kids:
                ports = [port] if recs[c][4] is None else recs[c][4]
                cname = name_of(nodes[c][0])
                srv += b"".join(srv_line(srvce, proto, name, srv_ttl(j), p, cname) for p in ports)
                n_srv += len(ports)
                if ports:
                    extra += a_line(cname, a_ttl(c), recs[c][2])
                    n_extra += 1
            add(SERVICE_SRV, j, srv, extra, n_srv, n_extra)
    return out
