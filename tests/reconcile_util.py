"""Independent restatement of regk_reconcile / regk_reconcile_requests, for the tests: a dictionary keyed by path
bytes, and the request frames from pyoracle's published jute layouts."""
from oracle import pyoracle

SAME, CREATE, UPDATE, DUP = 0, 1, 2, 3
KEEP, DELETE = 0, 1
NO_MATCH = 2 ** 64 - 1


class DuplicateNode(ValueError):
    def __init__(self, j):
        super().__init__("snapshot node %d repeats an earlier path" % j)
        self.index = j


def reconcile(paths, payloads, nodes):
    """paths / payloads of the desired records, nodes = [(path, data)] of the snapshot ->
    dict(cls, match, obs_cls, create, update, dup, delete)"""
    where = {}
    for j, (p, _) in enumerate(nodes):
        if p in where:
            raise DuplicateNode(j)
        where[p] = j
    first, cls, match = set(), [], []
    for p, d in zip(paths, payloads):
        j = where.get(p)
        match.append(NO_MATCH if j is None else j)
        if p in first:
            cls.append(DUP)
        elif j is None:
            cls.append(CREATE)
        else:
            cls.append(SAME if nodes[j][1] == d else UPDATE)
        first.add(p)
    obs_cls = [KEEP if p in first else DELETE for p, _ in nodes]
    pick = lambda c: [i for i, x in enumerate(cls) if x == c]
    return dict(cls=cls, match=match, obs_cls=obs_cls, create=pick(CREATE), update=pick(UPDATE), dup=pick(DUP),
                delete=[j for j, x in enumerate(obs_cls) if x == DELETE])


def frames(op, items, xid_base=1, group=0, zk_flags=1, version=-1):
    """regk_jute_requests' layout over [(path, data)]: one request per item (group 0) or multi transactions"""
    wrap = lambda x: (x + 2 ** 31) % 2 ** 32 - 2 ** 31
    if group == 0:
        return b"".join(pyoracle.jute_request(op, p, d, wrap(xid_base + k), zk_flags, version) for k, (p, d) in enumerate(items))
    return b"".join(pyoracle.jute_multi(op, items[k:k + group], wrap(xid_base + k // group), zk_flags, version)
                    for k in range(0, len(items), group))


def _murmur_step(h, w):
    w = (w * 0xCC9E2D51) & 0xFFFFFFFF
    w = ((w << 15) | (w >> 17)) & 0xFFFFFFFF
    w = (w * 0x1B873593) & 0xFFFFFFFF
    h ^= w
    h = ((h << 13) | (h >> 19)) & 0xFFFFFFFF
    return (h * 5 + 0xE6546B64) & 0xFFFFFFFF


def string_hash32(s: bytes) -> int:
    """string_hash32 of regk_core.cuh: murmur3 mixing over little-endian 4-byte groups, the last one zero-padded"""
    h = 0x9747B28C ^ len(s)
    for k in range(0, len(s), 4):
        h = _murmur_step(h, int.from_bytes(s[k:k + 4].ljust(4, b"\0"), "little"))
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & 0xFFFFFFFF
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & 0xFFFFFFFF
    return h ^ (h >> 16)
