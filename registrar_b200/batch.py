"""Struct-of-arrays batch of service records — the host-side image of
``regk_batch`` (include/regk.h).

One record carries exactly the inputs of the reference's per-record hot path:
``opts.domain`` (lib/register.js:205), ``os.hostname()`` (:222),
``registration.type`` / ``adminIp`` / ``registration.ttl`` /
``registration.ports`` (:141-151).  Citations are relative to /root/reference.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Iterable, List, Optional, Sequence

import numpy as np

TTL_ABSENT = -(2 ** 31)          # REGK_TTL_ABSENT

# README.md:274-282 — the host-record subtypes Binder understands.
README_TYPES = ["db_host", "host", "load_balancer", "moray_host", "ops_host", "redis_host", "rr_host"]

FLAG_IN_DEVICE = 1 << 0
FLAG_OUT_DEVICE = 1 << 1
FLAG_NODE_ALIAS = 1 << 2
FLAG_NO_JSON = 1 << 3
FLAG_NO_PATH = 1 << 4
FLAG_JOB_STEP = 1 << 5
FLAG_SKIP_BAD = 1 << 6           # skip out-of-domain records instead of refusing the batch (REGK_SKIP_BAD)

BAD_DOMAIN_BYTE = 1 << 0
BAD_HOST_BYTE = 1 << 1
BAD_ADDR_BYTE = 1 << 2
BAD_TYPE_ID = 1 << 3
BAD_TOO_LARGE = 1 << 4
BAD_SERVICE_BYTE = 1 << 5
BAD_KEY_ORDER = 1 << 6


def _pack(strings: Sequence[bytes]):
    off = np.zeros(len(strings) + 1, dtype=np.uint32)
    if strings:
        lens = np.fromiter((len(s) for s in strings), dtype=np.int64, count=len(strings))
        tot = int(lens.sum())
        if tot >= 2 ** 32:
            raise ValueError("packed field exceeds 4 GiB; split the batch")
        off[1:] = np.cumsum(lens)
    data = np.frombuffer(b"".join(strings), dtype=np.uint8).copy() if strings else np.zeros(0, np.uint8)
    return data, off


def _integral(v, lo: int, hi: int, what: str) -> int:
    """Numbers outside the kernels' domain are an error, never a silently different payload: the reference
    prints any JS number (ttl 1.5 -> "ttl":1.5, lib/register.js:144), the kernels print int32 / uint32."""
    if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or v != int(v):
        raise ValueError("%s %r is outside the supported input domain (integers only)" % (what, v))
    if not lo <= int(v) <= hi:
        raise ValueError("%s %r is outside the supported input domain [%d, %d]" % (what, v, lo, hi))
    return int(v)


def _b(x) -> bytes:
    return x if isinstance(x, (bytes, bytearray)) else str(x).encode("utf-8")


@dataclass
class RecordBatch:
    n: int
    types: List[bytes]
    domain_bytes: np.ndarray
    domain_off: np.ndarray
    host_bytes: np.ndarray
    host_off: Optional[np.ndarray]
    host_stride: int
    type_id: np.ndarray
    addr_bytes: np.ndarray
    addr_off: np.ndarray
    ttl: np.ndarray
    ports_off: Optional[np.ndarray]
    ports: Optional[np.ndarray]
    ports_present: Optional[np.ndarray] = None
    alias: bool = False
    meta: dict = field(default_factory=dict)

    # ---- construction -------------------------------------------------
    @classmethod
    def from_records(cls, records: Iterable[dict], types: Optional[Sequence] = None,
                     alias: bool = False) -> "RecordBatch":
        """records: dicts with keys domain, hostname (unless alias), type,
        address (adminIp), optional ttl (None = undefined), optional ports
        (None = undefined; [] is kept as an explicit empty array)."""
        records = list(records)
        tlist = [_b(t) for t in (types if types is not None else [])]
        tindex = {t: i for i, t in enumerate(tlist)}
        doms, hosts, addrs, tids, ttls, plist, present = [], [], [], [], [], [], []
        for r in records:
            doms.append(_b(r["domain"]))
            hosts.append(b"" if alias else _b(r["hostname"]))
            addrs.append(_b(r.get("address", r.get("adminIp", ""))))
            t = _b(r["type"])
            if t not in tindex:
                if types is not None:
                    raise KeyError("type %r not in the type table" % (t,))
                tindex[t] = len(tlist)
                tlist.append(t)
            tids.append(tindex[t])
            ttl = r.get("ttl")
            ttls.append(TTL_ABSENT if ttl is None else _integral(ttl, TTL_ABSENT + 1, 2 ** 31 - 1, "ttl"))
            p = r.get("ports")
            present.append(0 if p is None else 1)
            plist.append([] if p is None else [_integral(x, 0, 2 ** 32 - 1, "port") for x in p])
        if len(tlist) > 255:
            raise ValueError("at most 255 record types per batch")
        n = len(records)
        dbytes, doff = _pack(doms)
        abytes, aoff = _pack(addrs)
        hlens = {len(h) for h in hosts}
        if alias:
            hbytes, hoff, stride = np.zeros(0, np.uint8), None, 0
        elif len(hlens) == 1 and n > 0:
            hbytes, hoff, stride = np.frombuffer(b"".join(hosts), np.uint8).copy(), None, hlens.pop()
        else:
            hbytes, hoff = _pack(hosts)
            stride = 0
        poff = np.zeros(n + 1, dtype=np.uint32)
        if n:
            poff[1:] = np.cumsum([len(p) for p in plist])
        pflat = np.array([x for p in plist for x in p], dtype=np.uint32)
        pres = np.array(present, dtype=np.uint8)
        explicit_empty = any(pr and not p for pr, p in zip(present, plist))
        return cls(n=n, types=tlist, domain_bytes=dbytes, domain_off=doff, host_bytes=hbytes,
                   host_off=hoff, host_stride=stride, type_id=np.array(tids, dtype=np.uint8),
                   addr_bytes=abytes, addr_off=aoff, ttl=np.array(ttls, dtype=np.int32),
                   ports_off=poff, ports=pflat, ports_present=pres if explicit_empty else None,
                   alias=alias)

    # ---- views ----------------------------------------------------------
    def record(self, i: int) -> dict:
        d = bytes(self.domain_bytes[self.domain_off[i]:self.domain_off[i + 1]])
        if self.alias:
            h = b""
        elif self.host_off is not None:
            h = bytes(self.host_bytes[self.host_off[i]:self.host_off[i + 1]])
        else:
            h = bytes(self.host_bytes[i * self.host_stride:(i + 1) * self.host_stride])
        a = bytes(self.addr_bytes[self.addr_off[i]:self.addr_off[i + 1]])
        ttl = int(self.ttl[i])
        if self.ports_off is not None:
            p = [int(x) for x in self.ports[self.ports_off[i]:self.ports_off[i + 1]]]
        else:
            p = []
        present = bool(self.ports_present[i]) if self.ports_present is not None else len(p) > 0
        return {"domain": d, "hostname": h, "type": self.types[int(self.type_id[i])], "address": a,
                "ttl": None if ttl == TTL_ABSENT else ttl, "ports": p if present else None}

    def slice(self, lo: int, hi: int) -> "RecordBatch":
        """Records [lo, hi) as an independent batch (offsets rebased)."""
        def cut(data, off):
            o = off[lo:hi + 1].astype(np.int64)
            return data[o[0]:o[-1]].copy(), (o - o[0]).astype(np.uint32)
        db, do = cut(self.domain_bytes, self.domain_off)
        ab, ao = cut(self.addr_bytes, self.addr_off)
        if self.alias:
            hb, ho = self.host_bytes, None
        elif self.host_off is not None:
            hb, ho = cut(self.host_bytes, self.host_off)
        else:
            hb, ho = self.host_bytes[lo * self.host_stride:hi * self.host_stride].copy(), None
        if self.ports_off is not None:
            pb, po = cut(self.ports, self.ports_off)
        else:
            pb, po = None, None
        return RecordBatch(n=hi - lo, types=list(self.types), domain_bytes=db, domain_off=do,
                           host_bytes=hb, host_off=ho, host_stride=self.host_stride,
                           type_id=self.type_id[lo:hi].copy(), addr_bytes=ab, addr_off=ao,
                           ttl=self.ttl[lo:hi].copy(), ports_off=po, ports=pb,
                           ports_present=None if self.ports_present is None else self.ports_present[lo:hi].copy(),
                           alias=self.alias, meta=dict(self.meta))

    def take(self, indices) -> "RecordBatch":
        """The records at `indices` (in that order) as an independent batch, e.g. the records a skip-mode call
        skipped (HostResult.skipped), to be routed to another implementation."""
        idx = np.asarray(indices, dtype=np.int64).reshape(-1)
        if idx.size and (idx.min() < 0 or idx.max() >= self.n):
            raise IndexError("record index out of range [0, %d)" % self.n)

        def gather(data, off):
            o = off.astype(np.int64)
            lo = o[idx]
            lens = o[idx + 1] - lo
            noff = np.zeros(idx.size + 1, np.int64)
            np.cumsum(lens, out=noff[1:])
            pos = np.repeat(lo - noff[:-1], lens) + np.arange(int(noff[-1]), dtype=np.int64)
            return data[pos].copy(), noff.astype(np.uint32)
        db, do = gather(self.domain_bytes, self.domain_off)
        ab, ao = gather(self.addr_bytes, self.addr_off)
        if self.alias:
            hb, ho = self.host_bytes, None
        elif self.host_off is not None:
            hb, ho = gather(self.host_bytes, self.host_off)
        else:
            s = self.host_stride
            hb, ho = self.host_bytes[:self.n * s].reshape(self.n, s)[idx].reshape(-1).copy(), None
        if self.ports_off is not None:
            pb, po = gather(self.ports, self.ports_off)
        else:
            pb, po = None, None
        return RecordBatch(n=int(idx.size), types=list(self.types), domain_bytes=db, domain_off=do,
                           host_bytes=hb, host_off=ho, host_stride=self.host_stride,
                           type_id=self.type_id[idx].copy(), addr_bytes=ab, addr_off=ao,
                           ttl=self.ttl[idx].copy(), ports_off=po, ports=pb,
                           ports_present=None if self.ports_present is None else self.ports_present[idx].copy(),
                           alias=self.alias, meta=dict(self.meta))

    # ---- accounting (SURVEY.md §8d "algorithmic bytes per record") ----------
    def input_bytes(self) -> int:
        """B_in summed over the batch: L + 4 + H + len(addr) + 1 + 1 + 4 + 4 + 4k."""
        n = self.n
        dom = int(self.domain_off[-1])
        host = 0 if self.alias else (int(self.host_off[-1]) if self.host_off is not None else n * self.host_stride)
        addr = int(self.addr_off[-1])
        k = int(self.ports_off[-1]) if self.ports_off is not None else 0
        return dom + 4 * n + host + addr + n + n + 4 * n + 4 * n + 4 * k

    @staticmethod
    def output_bytes(path_total: int, json_total: int, n: int) -> int:
        """B_out summed: path bytes + payload bytes + two u64 offsets per record."""
        return path_total + json_total + 16 * n

    def h2d_bytes(self) -> int:
        """Bytes the library really copies host->device for this batch."""
        tot = 0
        for a in (self.domain_bytes, self.domain_off, self.host_bytes, self.host_off, self.type_id,
                  self.addr_bytes, self.addr_off, self.ttl, self.ports_off, self.ports, self.ports_present):
            if a is not None:
                tot += a.nbytes
        return tot


@dataclass
class Snapshot:
    """What a registry holds under the namespace a batch owns: m nodes, node j = (path j, data j), as u64 CSR streams
    (the layout regk_decode accepts).  Either all four arrays are host NumPy arrays (uint8 bytes, uint64 offsets) or
    all four are CUDA tensors (uint8 bytes, int64 offsets); a device snapshot's streams end at the byte tensors' ends.
    `version` / `owner` are each node's Stat.version (int32) and Stat.ephemeralOwner (int64, 0 = persistent), as the
    caller's client read them, on the same side as the streams; Context.reconcile_owned() needs them,
    Context.reconcile() ignores them.  Input of Context.reconcile() and Context.reconcile_owned()."""
    path_bytes: object
    path_off: object
    json_bytes: object
    json_off: object
    version: object = None
    owner: object = None

    @classmethod
    def from_nodes(cls, nodes: Iterable) -> "Snapshot":
        """[(path, data), ...] or [(path, data, version, owner), ...] -> host Snapshot"""
        nodes = list(nodes)
        stats = None
        arity = {len(x) for x in nodes}
        if len(arity) > 1 or not arity <= {2, 4}:
            raise ValueError("from_nodes takes (path, data) items or (path, data, version, owner) items, not a mix")
        if arity == {4}:
            stats = (np.array([x[2] for x in nodes], np.int32), np.array([x[3] for x in nodes], np.int64))
            nodes = [(x[0], x[1]) for x in nodes]

        def pack(strings):
            off = np.zeros(len(strings) + 1, np.uint64)
            if strings:
                np.cumsum([len(s) for s in strings], out=off[1:])
            return np.frombuffer(b"".join(strings), np.uint8).copy(), off
        pb, po = pack([_b(p) for p, _ in nodes])
        jb, jo = pack([_b(d) for _, d in nodes])
        return cls(pb, po, jb, jo) if stats is None else cls(pb, po, jb, jo, stats[0], stats[1])

    @property
    def device(self) -> bool:
        return hasattr(self.path_off, "data_ptr")

    @property
    def m(self) -> int:
        return (self.path_off.numel() if self.device else len(self.path_off)) - 1

    def cdecode_in(self):
        """regk_decode_in over the four arrays.  Returns (struct, keepalive)."""
        from ._native import CDecodeIn
        import ctypes as C
        if self.device:
            arrs = [self.path_bytes, self.path_off, self.json_bytes, self.json_off]
            if not all(a.is_cuda and a.is_contiguous() for a in arrs):
                raise ValueError("a device snapshot is four contiguous CUDA tensors")
            ptr = [a.data_ptr() or None for a in arrs]
            cin = CDecodeIn(n=self.m, flags=FLAG_IN_DEVICE, path_total=self.path_bytes.numel(),
                            json_total=self.json_bytes.numel(), path_bytes=ptr[0], path_off=ptr[1], json_bytes=ptr[2],
                            json_off=ptr[3])
            return cin, arrs
        keep = [np.ascontiguousarray(self.path_bytes, np.uint8), np.ascontiguousarray(self.path_off, np.uint64),
                np.ascontiguousarray(self.json_bytes, np.uint8), np.ascontiguousarray(self.json_off, np.uint64)]
        p = [a.ctypes.data_as(C.c_void_p) for a in keep]
        cin = CDecodeIn(n=len(keep[1]) - 1, flags=0, path_bytes=p[0], path_off=p[1], json_bytes=p[2], json_off=p[3])
        return cin, keep

    def cnode_stat(self, session: int, zk_flags: int):
        """regk_node_stat over `version` / `owner`.  Returns (struct, keepalive)."""
        from ._native import CNodeStat
        import ctypes as C
        if self.version is None or self.owner is None:
            raise ValueError("reconcile_owned needs the snapshot's version and owner arrays")
        m = self.m
        if self.device:
            import torch
            keep = [self.version, self.owner]
            if not all(a.is_cuda and a.is_contiguous() for a in keep):
                raise ValueError("a device snapshot's version and owner are contiguous CUDA tensors")
            if self.version.dtype != torch.int32 or self.owner.dtype != torch.int64:
                raise ValueError("a device snapshot's version is int32 and its owner int64, not %s / %s"
                                 % (self.version.dtype, self.owner.dtype))
            lens = (self.version.numel(), self.owner.numel())
            ptr = [a.data_ptr() or None for a in keep]
        else:
            keep = [np.asarray(self.version), np.asarray(self.owner)]
            if not all(a.dtype.kind in "iu" for a in keep):
                raise ValueError("version and owner are integer arrays")
            if (keep[0] != keep[0].astype(np.int32)).any() or (keep[1] != keep[1].astype(np.int64)).any():
                raise ValueError("a version outside int32 or an owner outside int64")
            keep = [np.ascontiguousarray(keep[0], np.int32), np.ascontiguousarray(keep[1], np.int64)]
            lens = (keep[0].size, keep[1].size)
            ptr = [a.ctypes.data_as(C.c_void_p) for a in keep]
        if lens != (m, m):
            raise ValueError("the snapshot has %d nodes but %d versions and %d owners" % (m, lens[0], lens[1]))
        return CNodeStat(version=ptr[0], ephemeral_owner=ptr[1], session=session, zk_flags=zk_flags), keep


SERVICE_KEYS = ("srvce", "proto", "port", "ttl")      # key ids 0..3 of regk_service_batch.key_order


@dataclass
class ServiceBatch:
    """Struct-of-arrays image of ``regk_service_batch``: one `registration.service` object per record
    (reference lib/register.js:186-199; the record written at :58-62)."""
    n: int
    srvce_bytes: np.ndarray
    srvce_off: np.ndarray
    proto_bytes: np.ndarray
    proto_off: np.ndarray
    port: np.ndarray
    ttl: np.ndarray
    key_order: Optional[np.ndarray] = None

    @classmethod
    def from_services(cls, services: Iterable[dict]) -> "ServiceBatch":
        """services: the callers' `registration.service` objects, {"type": "service", "service": {srvce, proto,
        port, ttl?}}.  The inner object's key order is kept (JSON.stringify follows insertion order); a missing
        ttl is defaulted to 60 and goes LAST, exactly what the assignment at lib/register.js:197 does."""
        services = list(services)
        srv, pro, ports, ttls, orders = [], [], [], [], []
        for i, s in enumerate(services):
            if list(s.keys()) != ["type", "service"] or s["type"] != "service":
                raise ValueError("service %d: expected {type: 'service', service: {...}} in that key order" % i)
            inner = s["service"]
            keys = list(inner.keys())
            extra = [k for k in keys if k not in SERVICE_KEYS]
            if extra:
                raise ValueError("service %d: members %r are outside the supported input domain" % (i, extra))
            for k in ("srvce", "proto", "port"):
                if k not in inner:
                    raise ValueError("service %d: %s is required" % (i, k))
            ttl = inner.get("ttl")
            if ttl is None:
                keys = [k for k in keys if k != "ttl"] + ["ttl"]
                ttl = 60
            srv.append(_b(inner["srvce"]))
            pro.append(_b(inner["proto"]))
            ports.append(_integral(inner["port"], 0, 2 ** 32 - 1, "service port"))
            ttls.append(_integral(ttl, -(2 ** 31), 2 ** 31 - 1, "service ttl"))
            orders.append(sum(SERVICE_KEYS.index(k) << (2 * j) for j, k in enumerate(keys)))
        sb, so = _pack(srv)
        pb, po = _pack(pro)
        return cls(n=len(services), srvce_bytes=sb, srvce_off=so, proto_bytes=pb, proto_off=po,
                   port=np.array(ports, np.uint32), ttl=np.array(ttls, np.int32), key_order=np.array(orders, np.uint8))
