"""ctypes binding of libregk.so (include/regk.h).

This is the only way record bytes are produced in this package: every call
goes through the C-ABI into the sm_90a kernels.  There is deliberately no
Python/NumPy implementation of the path here — if the shared library is not
built, or no CUDA device is usable, the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

from .batch import (FLAG_IN_DEVICE, FLAG_JOB_STEP, FLAG_NODE_ALIAS, FLAG_NO_JSON, FLAG_NO_PATH, FLAG_OUT_DEVICE,
                    FLAG_SKIP_BAD, RecordBatch)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("REGK_LIB") or os.path.join(_HERE, "libregk.so")      # REGK_LIB: A/B builds (dev)

REGK_OK = 0
REGK_ERR_INVALID_ARG = 1
REGK_ERR_CUDA = 2
REGK_ERR_OUT_OF_DOMAIN = 3
REGK_ERR_NOMEM = 4
REGK_ERR_STATE = 5


class RegkError(RuntimeError):
    def __init__(self, code: int, message: str, result=None):
        super().__init__("regk error %d: %s" % (code, message))
        self.code = code
        self.message = message
        self.result = result


class OutOfDomainError(RegkError):
    """A record is outside the fenced input domain (REGK_ERR_OUT_OF_DOMAIN)."""


class CBatch(C.Structure):           # regk_batch
    _fields_ = [("n", C.c_uint64), ("flags", C.c_uint32), ("host_stride", C.c_uint32),
                ("domain_bytes_len", C.c_uint64), ("host_bytes_len", C.c_uint64),
                ("addr_bytes_len", C.c_uint64), ("ports_len", C.c_uint64),
                ("domain_bytes", C.c_void_p), ("domain_off", C.c_void_p),
                ("host_bytes", C.c_void_p), ("host_off", C.c_void_p),
                ("type_id", C.c_void_p),
                ("addr_bytes", C.c_void_p), ("addr_off", C.c_void_p),
                ("ttl", C.c_void_p),
                ("ports_off", C.c_void_p), ("ports", C.c_void_p), ("ports_present", C.c_void_p)]


class CResult(C.Structure):          # regk_result
    _fields_ = [("n", C.c_uint64), ("flags", C.c_uint32), ("bad_bits", C.c_uint32),
                ("first_bad", C.c_uint64),
                ("path_bytes", C.c_void_p), ("path_off", C.c_void_p), ("path_total", C.c_uint64),
                ("json_bytes", C.c_void_p), ("json_off", C.c_void_p), ("json_total", C.c_uint64),
                ("kernel_ms", C.c_float), ("path_kernel_ms", C.c_float), ("json_kernel_ms", C.c_float),
                ("json_len_kernel_ms", C.c_float), ("launches", C.c_uint32), ("opaque", C.c_void_p),
                ("job_path_base", C.c_uint64), ("job_path_total", C.c_uint64),
                ("job_json_base", C.c_uint64), ("job_json_total", C.c_uint64),
                ("generic_tiles", C.c_uint32), ("reserved", C.c_uint32),
                ("path_off32", C.c_void_p), ("json_off32", C.c_void_p)]


MAX_PEERS = 16
IPC_HANDLE_BYTES = 64


class CGather(C.Structure):          # regk_gather
    _fields_ = [("world", C.c_uint32), ("rank", C.c_uint32), ("rec_base", C.c_uint64), ("n_total", C.c_uint64),
                ("totals", C.c_void_p),
                ("path_bytes", C.c_void_p * MAX_PEERS), ("path_off", C.c_void_p * MAX_PEERS),
                ("json_bytes", C.c_void_p * MAX_PEERS), ("json_off", C.c_void_p * MAX_PEERS),
                ("path_cap", C.c_uint64), ("json_cap", C.c_uint64)]


class CServiceBatch(C.Structure):    # regk_service_batch
    _fields_ = [("n", C.c_uint64), ("flags", C.c_uint32), ("reserved", C.c_uint32),
                ("srvce_bytes_len", C.c_uint64), ("proto_bytes_len", C.c_uint64),
                ("srvce_bytes", C.c_void_p), ("srvce_off", C.c_void_p),
                ("proto_bytes", C.c_void_p), ("proto_off", C.c_void_p),
                ("port", C.c_void_p), ("ttl", C.c_void_p), ("key_order", C.c_void_p)]


class CFrames(C.Structure):          # regk_frames
    _fields_ = [("n", C.c_uint64), ("total", C.c_uint64), ("flags", C.c_uint32), ("launches", C.c_uint32),
                ("frame_bytes", C.c_void_p), ("frame_off", C.c_void_p), ("kernel_ms", C.c_float)]


class CJuteOpts(C.Structure):        # regk_jute_opts
    _fields_ = [("op", C.c_uint32), ("flags", C.c_uint32), ("xid_base", C.c_int32), ("zk_flags", C.c_uint32),
                ("version", C.c_int32), ("group", C.c_uint32)]


ZK_CREATE, ZK_DELETE, ZK_SETDATA = 1, 2, 5
ZK_GETDATA = 4                      # jute_requests: GetDataRequest{path, watch = false}; its replies go to read_replies()
ZK_REPLACE = 256                    # reconcile_requests after reconcile_owned: delete + create in one multi transaction
FLAG_ZK_VERSION_OBSERVED = 1 << 9   # regk_jute_opts.flags: each frame carries its node's Stat.version


class CDecodeIn(C.Structure):        # regk_decode_in
    _fields_ = [("n", C.c_uint64), ("flags", C.c_uint32), ("host_nodes", C.c_uint32),
                ("path_total", C.c_uint64), ("json_total", C.c_uint64),
                ("path_bytes", C.c_void_p), ("path_off", C.c_void_p), ("json_bytes", C.c_void_p), ("json_off", C.c_void_p)]


class CDecodeOut(C.Structure):       # regk_decode_out
    _fields_ = [("n", C.c_uint64), ("flags", C.c_uint32), ("launches", C.c_uint32),
                ("rec", C.c_void_p), ("dom_bytes", C.c_void_p), ("ports", C.c_void_p),
                ("dom_bytes_len", C.c_uint64), ("ports_len", C.c_uint64), ("kernel_ms", C.c_float)]


# regk_decoded as a NumPy record type
DECODED_DTYPE = np.dtype([("flags", "<u4"), ("dom_len", "<u4"), ("host_pos", "<u4"), ("host_len", "<u4"),
                          ("type_pos", "<u4"), ("type_len", "<u4"), ("addr_pos", "<u4"), ("addr_len", "<u4"),
                          ("ttl", "<i4"), ("nports", "<u4")])
FLAG_DECODE_LAST = 1 << 8
DEC_PATH_OK, DEC_HOST_RECORD, DEC_SERVICE_RECORD, DEC_NOT_CANONICAL = 1, 2, 4, 8
DEC_KEY_MISMATCH, DEC_ADDR_MISMATCH, DEC_BAD_NUMBER, DEC_BAD_PATH = 16, 32, 64, 128

MAILBOX_BYTES = MAX_PEERS * 32


class CJob(C.Structure):             # regk_job
    _fields_ = [("world", C.c_uint32), ("rank", C.c_uint32), ("rec_base", C.c_uint64), ("n_total", C.c_uint64),
                ("path_bytes", C.c_void_p * MAX_PEERS), ("path_off", C.c_void_p * MAX_PEERS),
                ("json_bytes", C.c_void_p * MAX_PEERS), ("json_off", C.c_void_p * MAX_PEERS),
                ("mailbox", C.c_void_p * MAX_PEERS),
                ("path_cap", C.c_uint64), ("json_cap", C.c_uint64), ("timeout_ms", C.c_uint64)]


class CParents(C.Structure):         # regk_parents
    _fields_ = [("n", C.c_uint64), ("n_unique", C.c_uint64), ("flags", C.c_uint32), ("launches", C.c_uint32),
                ("parent_len", C.c_void_p), ("unique_first", C.c_void_p), ("kernel_ms", C.c_float)]


class CDirs(C.Structure):            # regk_dirs
    _fields_ = [("n", C.c_uint64), ("n_dirs", C.c_uint64), ("n_invalid", C.c_uint64), ("flags", C.c_uint32),
                ("launches", C.c_uint32), ("max_depth", C.c_uint32), ("reserved", C.c_uint32),
                ("dir_rec", C.c_void_p), ("dir_len", C.c_void_p), ("depth_off", C.c_void_p), ("dir_bytes", C.c_void_p),
                ("dir_off", C.c_void_p), ("invalid", C.c_void_p), ("dir_bytes_len", C.c_uint64),
                ("kernel_ms", C.c_float), ("parent_ms", C.c_float), ("closure_ms", C.c_float), ("gather_ms", C.c_float)]


class DirSet:
    """Host copy of a regk_dirs: the directories register() must create for a batch, parents first.  Directory k is
    dir_bytes[dir_off[k]:dir_off[k+1]] == path(dir_rec[k])[:dir_len[k]]; depth d is directories
    depth_off[d-1]:depth_off[d]; `invalid` lists the first record of every directory ZooKeeper would reject."""

    def __init__(self, out):
        nd, ni = int(out.n_dirs), int(out.n_invalid)
        self.n, self.n_dirs, self.max_depth, self.launches = int(out.n), nd, int(out.max_depth), int(out.launches)
        self.dir_rec = _as_np(out.dir_rec, nd, np.uint64).copy()
        self.dir_len = _as_np(out.dir_len, nd, np.uint32).copy()
        self.depth_off = _as_np(out.depth_off, self.max_depth + 1, np.uint64).copy()
        self.dir_bytes = _as_np(out.dir_bytes, int(out.dir_bytes_len), np.uint8).copy()
        self.dir_off = _as_np(out.dir_off, nd + 1, np.uint64).copy()
        self.invalid = _as_np(out.invalid, ni, np.uint64).copy()
        self.kernel_ms, self.parent_ms = float(out.kernel_ms), float(out.parent_ms)
        self.closure_ms, self.gather_ms = float(out.closure_ms), float(out.gather_ms)

    def dirs(self):
        b = self.dir_bytes.tobytes()
        return [b[int(self.dir_off[k]):int(self.dir_off[k + 1])] for k in range(self.n_dirs)]


class CDelta(C.Structure):           # regk_delta
    _fields_ = [("n", C.c_uint64), ("m", C.c_uint64), ("n_same", C.c_uint64), ("n_create", C.c_uint64),
                ("n_update", C.c_uint64), ("n_dup", C.c_uint64), ("n_delete", C.c_uint64),
                ("flags", C.c_uint32), ("launches", C.c_uint32),
                ("cls", C.c_void_p), ("match", C.c_void_p), ("obs_cls", C.c_void_p),
                ("create", C.c_void_p), ("update", C.c_void_p), ("dup", C.c_void_p), ("del_", C.c_void_p),
                ("kernel_ms", C.c_float)]


DELTA_SAME, DELTA_CREATE, DELTA_UPDATE, DELTA_DUP = 0, 1, 2, 3       # Delta.cls
DELTA_REPLACE = 4                                                    # Delta.cls, reconcile_owned only
DELTA_KEEP, DELTA_DELETE = 0, 1                                      # Delta.obs_cls


class Delta:
    """Host copy of a regk_delta: how the batch finished last differs from a snapshot of the registry.  cls[i] is
    DELTA_SAME / _CREATE / _UPDATE / _DUP for record i, match[i] the snapshot node with its path (UINT64_MAX: none),
    obs_cls[j] DELTA_KEEP / _DELETE for node j; create / update / dup are ascending record indices, delete ascending
    snapshot indices.  From reconcile_owned, cls may also hold DELTA_REPLACE and `replace` lists those records
    (ascending); a plain reconcile reports n_replace == 0."""

    def __init__(self, out, replace=None, n_replace=0):
        n, m = int(out.n), int(out.m)
        self.n, self.m, self.launches, self.kernel_ms = n, m, int(out.launches), float(out.kernel_ms)
        self.n_same, self.n_create, self.n_update = int(out.n_same), int(out.n_create), int(out.n_update)
        self.n_dup, self.n_delete = int(out.n_dup), int(out.n_delete)
        self.cls = _as_np(out.cls, n, np.uint8).copy()
        self.match = _as_np(out.match, n, np.uint64).copy()
        self.obs_cls = _as_np(out.obs_cls, m, np.uint8).copy()
        self.create = _as_np(out.create, self.n_create, np.uint64).copy()
        self.update = _as_np(out.update, self.n_update, np.uint64).copy()
        self.dup = _as_np(out.dup, self.n_dup, np.uint64).copy()
        self.delete = _as_np(out.del_, self.n_delete, np.uint64).copy()
        self.n_replace = int(n_replace)
        self.replace = _as_np(replace, self.n_replace, np.uint64).copy()


class CNodeStat(C.Structure):        # regk_node_stat
    _fields_ = [("version", C.c_void_p), ("ephemeral_owner", C.c_void_p), ("session", C.c_int64),
                ("zk_flags", C.c_uint32), ("reserved", C.c_uint32)]


class CDeltaOwned(C.Structure):      # regk_delta_owned
    _fields_ = [("d", CDelta), ("n_replace", C.c_uint64), ("replace", C.c_void_p)]


class CReplies(C.Structure):        # regk_replies
    _fields_ = [("n", C.c_uint64), ("m", C.c_uint64), ("n_found", C.c_uint64), ("n_missing", C.c_uint64),
                ("n_error", C.c_uint64), ("n_skipped", C.c_uint64), ("consumed", C.c_uint64),
                ("flags", C.c_uint32), ("launches", C.c_uint32), ("err", C.c_void_p), ("node_rec", C.c_void_p),
                ("snapshot", CDecodeIn), ("version", C.c_void_p), ("ephemeral_owner", C.c_void_p),
                ("kernel_ms", C.c_float)]


class Replies:
    """What read_replies() made of the replies to the last getData framing: err[k] is the ReplyHeader.err of record
    k's reply (0 found, -101 NONODE, other codes), node_rec[j] the record whose reply gave snapshot node j (ascending,
    one node per distinct path among the found replies), plus n_found / n_missing / n_error / n_skipped and `consumed`
    (stream bytes up to the end of the n-th reply).  The snapshot itself stays on the device: pass this object to
    Context.reconcile_owned(replies, session=..., zk_flags=...) as it is, or copy it out with snapshot().  A record whose
    reply carries an error other than NONODE gets no node either, so reconcile classes it CREATE: do not send the repair
    while n_error > 0.  The snapshot is valid until the next read_replies() call on the context."""

    def __init__(self, ctx, out):
        self._ctx, self._out = ctx, out
        n, m = int(out.n), int(out.m)
        self.n, self.m, self.launches, self.kernel_ms = n, m, int(out.launches), float(out.kernel_ms)
        self.n_found, self.n_missing, self.n_error = int(out.n_found), int(out.n_missing), int(out.n_error)
        self.n_skipped, self.consumed = int(out.n_skipped), int(out.consumed)
        self.err = _as_np(out.err, n, np.int32).copy()
        self.node_rec = _as_np(out.node_rec, m, np.uint64).copy()

    def cdecode_in(self):
        """the device regk_decode_in of the snapshot.  Returns (struct, keepalive)."""
        return self._out.snapshot, None

    def cnode_stat(self, session: int, zk_flags: int):
        """regk_node_stat over the snapshot's device version / owner arrays.  Returns (struct, keepalive)."""
        return CNodeStat(version=self._out.version, ephemeral_owner=self._out.ephemeral_owner, session=session,
                         zk_flags=zk_flags), None

    def snapshot(self):
        """host batch.Snapshot copy of the snapshot, with version and owner"""
        from .batch import Snapshot
        s, m = self._out.snapshot, self.m
        d2h = lambda ptr, count, dtype: self._ctx._d2h(ptr, count, dtype)
        return Snapshot(d2h(s.path_bytes, int(s.path_total), np.uint8), d2h(s.path_off, m + 1, np.uint64),
                        d2h(s.json_bytes, int(s.json_total), np.uint8), d2h(s.json_off, m + 1, np.uint64),
                        d2h(self._out.version, m, np.int32), d2h(self._out.ephemeral_owner, m, np.int64))


class CSkipped(C.Structure):         # regk_skipped
    _fields_ = [("n", C.c_uint64), ("n_skipped", C.c_uint64), ("flags", C.c_uint32), ("bad_bits", C.c_uint32),
                ("index", C.c_void_p), ("bits", C.c_void_p)]


EXPORTS = ["regk_abi_version", "regk_create", "regk_destroy", "regk_last_error", "regk_set_stream",
           "regk_set_types", "regk_register_batch", "regk_finish", "regk_release", "regk_host_alloc",
           "regk_host_free", "regk_dev_alloc", "regk_dev_free", "regk_memcpy_h2d", "regk_memcpy_d2h",
           "regk_sync", "regk_set_option", "regk_get_option", "regk_ipc_export", "regk_ipc_open", "regk_ipc_close",
           "regk_gather_push", "regk_parent_dirs", "regk_job_bind", "regk_service_records",
           "regk_jute_frames", "regk_jute_requests", "regk_decode", "regk_skipped_records", "regk_mkdirp_dirs",
           "regk_mkdirp_requests", "regk_reconcile", "regk_reconcile_requests", "regk_reconcile_owned",
           "regk_read_replies"]

_lib = None


def load_library():
    """dlopen libregk.so and type its entry points; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "registrar_b200: %s is missing — build it with `python -c 'import __graft_entry__ as g; g.build()'`. "
            "There is no CPU fallback for the registration path." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, u32, u64, i64, sz = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int64, C.c_size_t
    lib.regk_abi_version.restype = C.c_int
    lib.regk_create.argtypes = [C.c_int, C.POINTER(vp)]
    lib.regk_destroy.argtypes = [vp]
    lib.regk_destroy.restype = None
    lib.regk_last_error.argtypes = [vp]
    lib.regk_last_error.restype = C.c_char_p
    lib.regk_set_stream.argtypes = [vp, vp]
    lib.regk_set_types.argtypes = [vp, C.POINTER(C.c_char_p), C.POINTER(u32), u32]
    lib.regk_register_batch.argtypes = [vp, C.POINTER(CBatch), C.POINTER(CResult)]
    lib.regk_finish.argtypes = [vp, C.POINTER(CResult)]
    lib.regk_release.argtypes = [vp, C.POINTER(CResult)]
    lib.regk_host_alloc.argtypes = [vp, sz]
    lib.regk_host_alloc.restype = vp
    lib.regk_host_free.argtypes = [vp, vp]
    lib.regk_host_free.restype = None
    lib.regk_dev_alloc.argtypes = [vp, sz]
    lib.regk_dev_alloc.restype = vp
    lib.regk_dev_free.argtypes = [vp, vp]
    lib.regk_dev_free.restype = None
    lib.regk_memcpy_h2d.argtypes = [vp, vp, vp, sz]
    lib.regk_memcpy_d2h.argtypes = [vp, vp, vp, sz]
    lib.regk_sync.argtypes = [vp]
    lib.regk_set_option.argtypes = [vp, C.c_char_p, i64]
    lib.regk_get_option.argtypes = [vp, C.c_char_p]
    lib.regk_get_option.restype = i64
    lib.regk_ipc_export.argtypes = [vp, vp, C.c_char_p]
    lib.regk_ipc_open.argtypes = [vp, C.c_char_p, C.POINTER(vp)]
    lib.regk_ipc_close.argtypes = [vp, vp]
    lib.regk_gather_push.argtypes = [vp, C.POINTER(CResult), C.POINTER(CGather)]
    lib.regk_parent_dirs.argtypes = [vp, u32, C.POINTER(CParents)]
    lib.regk_job_bind.argtypes = [vp, C.POINTER(CJob)]
    lib.regk_service_records.argtypes = [vp, C.POINTER(CServiceBatch), C.POINTER(CResult)]
    lib.regk_jute_frames.argtypes = [vp, u32, C.c_int32, u32, C.POINTER(CFrames)]
    lib.regk_jute_requests.argtypes = [vp, C.POINTER(CJuteOpts), C.POINTER(CFrames)]
    lib.regk_decode.argtypes = [vp, C.POINTER(CDecodeIn), C.POINTER(CDecodeOut)]
    lib.regk_skipped_records.argtypes = [vp, u32, C.POINTER(CSkipped)]
    lib.regk_mkdirp_dirs.argtypes = [vp, u32, C.POINTER(CDirs)]
    lib.regk_mkdirp_requests.argtypes = [vp, C.c_int32, u32, u32, C.POINTER(CFrames)]
    lib.regk_reconcile.argtypes = [vp, C.POINTER(CDecodeIn), u32, C.POINTER(CDelta)]
    lib.regk_reconcile_requests.argtypes = [vp, C.POINTER(CJuteOpts), C.POINTER(CFrames)]
    lib.regk_reconcile_owned.argtypes = [vp, C.POINTER(CDecodeIn), C.POINTER(CNodeStat), u32, C.POINTER(CDeltaOwned)]
    lib.regk_read_replies.argtypes = [vp, vp, u64, u32, C.POINTER(CReplies)]
    _lib = lib
    return lib


def _np_ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def host_cbatch(b: RecordBatch, flags: int = 0):
    """regk_batch over the NumPy arrays of a host RecordBatch.  Returns (struct, keepalive)."""
    keep = [None if x is None else np.ascontiguousarray(x) for x in (
        b.domain_bytes, b.domain_off, b.host_bytes, b.host_off, b.type_id, b.addr_bytes, b.addr_off, b.ttl,
        b.ports_off, b.ports, b.ports_present)]
    n = b.n
    cb = CBatch(
        n=n, flags=flags | (FLAG_NODE_ALIAS if b.alias else 0), host_stride=b.host_stride,
        domain_bytes_len=int(b.domain_off[-1]) if n else 0,
        host_bytes_len=0 if b.alias else (int(b.host_off[-1]) if b.host_off is not None else n * b.host_stride),
        addr_bytes_len=int(b.addr_off[-1]) if n else 0,
        ports_len=int(b.ports_off[-1]) if (b.ports_off is not None and n) else 0,
        domain_bytes=_np_ptr(keep[0]), domain_off=_np_ptr(keep[1]), host_bytes=_np_ptr(keep[2]),
        host_off=_np_ptr(keep[3]), type_id=_np_ptr(keep[4]), addr_bytes=_np_ptr(keep[5]),
        addr_off=_np_ptr(keep[6]), ttl=_np_ptr(keep[7]), ports_off=_np_ptr(keep[8]), ports=_np_ptr(keep[9]),
        ports_present=_np_ptr(keep[10]))
    return cb, keep


class HostResult:
    """Host copy of a regk_result (NumPy views are copied out of the library's pinned buffers
    unless copy=False).  A skip-mode result also carries `skipped` (uint64, ascending record indices) and
    `skipped_bits` (uint8, REGK_BAD_* of each); those records have empty paths and payloads."""

    def __init__(self, n, path_bytes, path_off, json_bytes, json_off, kernel_ms, path_ms, json_ms, launches,
                 json_len_ms=0.0, generic_tiles=0):
        self.generic_tiles = generic_tiles
        self.skipped = None
        self.skipped_bits = None
        self.n = n
        self.path_bytes, self.path_off = path_bytes, path_off
        self.json_bytes, self.json_off = json_bytes, json_off
        self.kernel_ms, self.path_kernel_ms, self.json_kernel_ms = kernel_ms, path_ms, json_ms
        self.json_len_kernel_ms = json_len_ms
        self.launches = launches

    @property
    def path_total(self):
        return int(self.path_off[-1])

    @property
    def json_total(self):
        return int(self.json_off[-1])

    def path(self, i: int) -> bytes:
        return bytes(self.path_bytes[int(self.path_off[i]):int(self.path_off[i + 1])])

    def json(self, i: int) -> bytes:
        return bytes(self.json_bytes[int(self.json_off[i]):int(self.json_off[i + 1])])


def _offsets(res, which: str, n: int):
    """The offset array of a finished host result: uint64, or uint32 under option "offsets32"."""
    p32 = getattr(res, which + "32")
    return _as_np(p32, n + 1, np.uint32) if p32 else _as_np(getattr(res, which), n + 1, np.uint64)


def _as_np(ptr, count, dtype):
    if count == 0 or not ptr:
        return np.zeros(0, dtype)
    buf = (C.c_uint8 * (count * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=count)


class Context:
    """One regk_ctx: one CUDA device, one stream, single owner thread."""

    def __init__(self, device: int = 0, types=None):
        self._lib = load_library()
        h = C.c_void_p()
        rc = self._lib.regk_create(device, C.byref(h))
        if rc != REGK_OK:
            raise RegkError(rc, (self._lib.regk_last_error(None) or b"").decode())
        self._h = h
        self.device = device
        self._types = None
        if types is not None:
            self.set_types(types)

    # -- lifecycle --
    def close(self):
        if getattr(self, "_h", None):
            self._lib.regk_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self) -> str:
        return (self._lib.regk_last_error(self._h) or b"").decode()

    def _check(self, rc, result=None):
        if rc == REGK_OK:
            return
        cls = OutOfDomainError if rc == REGK_ERR_OUT_OF_DOMAIN else RegkError
        raise cls(rc, self._err(), result)

    # -- configuration --
    def set_types(self, types):
        tl = [t if isinstance(t, (bytes, bytearray)) else str(t).encode("utf-8") for t in types]
        if self._types == tl:
            return
        arr = (C.c_char_p * max(len(tl), 1))(*tl)
        lens = (C.c_uint32 * max(len(tl), 1))(*[len(t) for t in tl])
        self._check(self._lib.regk_set_types(self._h, arr, lens, len(tl)))
        self._types = tl

    def set_option(self, name: str, value: int):
        self._check(self._lib.regk_set_option(self._h, name.encode(), int(value)))

    def get_option(self, name: str) -> int:
        return int(self._lib.regk_get_option(self._h, name.encode()))

    def set_stream(self, cuda_stream: int):
        """Run on the caller's CUDA stream (a cudaStream_t as an integer, e.g. torch's stream.cuda_stream).
        torch reports the legacy default stream as 0, which the C-ABI reads as "the library's own stream":
        0 is therefore passed on as cudaStreamLegacy (0x1), so that the caller's events, NCCL calls and the
        library's kernels really are in one stream order.  Use set_own_stream() for the library's stream."""
        self._check(self._lib.regk_set_stream(self._h, C.c_void_p(cuda_stream if cuda_stream else 1)))

    def set_own_stream(self):
        self._check(self._lib.regk_set_stream(self._h, None))

    def sync(self):
        self._check(self._lib.regk_sync(self._h))

    # -- the hot path, host buffers in / host buffers out --
    def register_batch(self, batch: RecordBatch, paths: bool = True, payloads: bool = True,
                       copy: bool = True, skip_bad: bool = False) -> HostResult:
        """Host RecordBatch -> HostResult through regk_register_batch (H2D, kernels, D2H).  skip_bad=True: records
        outside the fenced input domain come back empty and are listed in result.skipped instead of refusing the
        batch (REGK_SKIP_BAD)."""
        self.set_types(batch.types)
        flags = (0 if paths else FLAG_NO_PATH) | (0 if payloads else FLAG_NO_JSON) | (FLAG_SKIP_BAD if skip_bad else 0)
        cb, keep = host_cbatch(batch, flags)
        res = CResult()
        rc = self._lib.regk_register_batch(self._h, C.byref(cb), C.byref(res))
        del keep
        if rc != REGK_OK:
            self._check(rc, res)
        n = int(res.n)
        cp = (lambda a: a.copy()) if copy else (lambda a: a)
        out = HostResult(
            n, cp(_as_np(res.path_bytes, int(res.path_total), np.uint8)), cp(_offsets(res, "path_off", n)),
            cp(_as_np(res.json_bytes, int(res.json_total), np.uint8)), cp(_offsets(res, "json_off", n)),
            float(res.kernel_ms), float(res.path_kernel_ms), float(res.json_kernel_ms), int(res.launches),
            float(res.json_len_kernel_ms), int(res.generic_tiles))
        if skip_bad:
            out.skipped, out.skipped_bits = self.skipped_records()
        self._lib.regk_release(self._h, C.byref(res))
        return out

    def skipped_records(self, device: bool = False):
        """(index uint64[n_skipped], bad_bits uint8[n_skipped]) of the skip-mode batch finished last on this
        context (regk_skipped_records).  device=True returns the raw CSkipped (device pointers)."""
        out = CSkipped()
        self._check(self._lib.regk_skipped_records(self._h, FLAG_OUT_DEVICE if device else 0, C.byref(out)))
        if device:
            return out
        k = int(out.n_skipped)
        return _as_np(out.index, k, np.uint64).copy(), _as_np(out.bits, k, np.uint8).copy()

    # -- service records (lib/register.js:45-75), host buffers in / host buffers out --
    def service_records(self, sb) -> HostResult:
        """ServiceBatch -> payloads of the persistent service nodes (only json_* of the result are filled)."""
        keep = [None if x is None else np.ascontiguousarray(x) for x in (
            sb.srvce_bytes, sb.srvce_off, sb.proto_bytes, sb.proto_off, sb.port, sb.ttl, sb.key_order)]
        n = sb.n
        cb = CServiceBatch(n=n, flags=0, srvce_bytes_len=int(sb.srvce_off[-1]) if n else 0,
                           proto_bytes_len=int(sb.proto_off[-1]) if n else 0,
                           srvce_bytes=_np_ptr(keep[0]), srvce_off=_np_ptr(keep[1]), proto_bytes=_np_ptr(keep[2]),
                           proto_off=_np_ptr(keep[3]), port=_np_ptr(keep[4]), ttl=_np_ptr(keep[5]),
                           key_order=_np_ptr(keep[6]))
        res = CResult()
        rc = self._lib.regk_service_records(self._h, C.byref(cb), C.byref(res))
        del keep
        if rc != REGK_OK:
            self._check(rc, res)
        out = HostResult(n, np.zeros(0, np.uint8), np.zeros(n + 1, np.uint64),
                         _as_np(res.json_bytes, int(res.json_total), np.uint8).copy(),
                         _as_np(res.json_off, n + 1, np.uint64).copy(), float(res.kernel_ms), 0.0,
                         float(res.json_kernel_ms), int(res.launches))
        self._lib.regk_release(self._h, C.byref(res))
        return out

    # -- ZooKeeper wire frames of the batch finished last (lib/register.js:156-159 -> zkplus -> jute) --
    def jute_frames(self, xid_base: int = 1, zk_flags: int = 1, device: bool = False):
        """(frame_bytes uint8[total], frame_off uint64[n+1], kernel_ms): one CreateRequest per record of the batch
        finished last on this context.  device=True returns the raw CFrames (device pointers)."""
        out = CFrames()
        self._check(self._lib.regk_jute_frames(self._h, FLAG_OUT_DEVICE if device else 0, int(xid_base), int(zk_flags),
                                               C.byref(out)))
        if device:
            return out
        n = int(out.n)
        return (_as_np(out.frame_bytes, int(out.total), np.uint8).copy(), _as_np(out.frame_off, n + 1, np.uint64).copy(),
                float(out.kernel_ms))

    def jute_requests(self, op: int = ZK_CREATE, xid_base: int = 1, zk_flags: int = 1, version: int = -1, group: int = 0,
                      device: bool = False):
        """regk_jute_requests: create / delete / setData requests of the batch finished last, one per record
        (group=0) or as multi transactions of `group` operations.  Returns (frame_bytes, frame_off uint64[frames+1],
        kernel_ms), or the raw CFrames with device=True."""
        o = CJuteOpts(int(op), FLAG_OUT_DEVICE if device else 0, int(xid_base), int(zk_flags), int(version), int(group))
        out = CFrames()
        self._check(self._lib.regk_jute_requests(self._h, C.byref(o), C.byref(out)))
        if device:
            return out
        n = int(out.n)
        return (_as_np(out.frame_bytes, int(out.total), np.uint8).copy(), _as_np(out.frame_off, n + 1, np.uint64).copy(),
                float(out.kernel_ms))

    # -- the reader side: paths and payloads back into records --
    def decode(self, path_bytes=None, path_off=None, json_bytes=None, json_off=None, host_nodes: bool = True,
               last: bool = False):
        """regk_decode over explicit host streams (uint8 bytes + uint64 CSR offsets) or, with last=True, over the
        batch finished last on this context.  Returns (rec: structured array of regk_decoded, dom_bytes in slot
        layout, ports in slot layout, kernel_ms)."""
        keep = [None if path_bytes is None else np.ascontiguousarray(path_bytes, dtype=np.uint8),
                None if path_off is None else np.ascontiguousarray(path_off, dtype=np.uint64),    # also accepts 32-bit offsets
                None if json_bytes is None else np.ascontiguousarray(json_bytes, dtype=np.uint8),
                None if json_off is None else np.ascontiguousarray(json_off, dtype=np.uint64)]
        n = 0
        for off in (keep[1], keep[3]):
            if off is not None:
                n = len(off) - 1
        cin = CDecodeIn(n=n, flags=FLAG_DECODE_LAST if last else 0, host_nodes=1 if host_nodes else 0,
                        path_bytes=_np_ptr(keep[0]), path_off=_np_ptr(keep[1]), json_bytes=_np_ptr(keep[2]),
                        json_off=_np_ptr(keep[3]))
        out = CDecodeOut()
        self._check(self._lib.regk_decode(self._h, C.byref(cin), C.byref(out)))
        n = int(out.n)
        rec = np.frombuffer((C.c_uint8 * (n * DECODED_DTYPE.itemsize)).from_address(out.rec), dtype=DECODED_DTYPE,
                            count=n).copy() if n else np.zeros(0, DECODED_DTYPE)
        return (rec, _as_np(out.dom_bytes, int(out.dom_bytes_len), np.uint8).copy(),
                _as_np(out.ports, int(out.ports_len), np.uint32).copy(), float(out.kernel_ms))

    # -- two-deep submission of host batches: the next batch's H2D overlaps this batch's result traffic --
    def submit(self, batch: RecordBatch, paths: bool = True, payloads: bool = True, skip_bad: bool = False):
        """Enqueue a host RecordBatch and return a ticket for collect().  Needs set_option("async", 1); the
        batch's arrays must stay alive and unchanged until collect().  At most two tickets may be open."""
        self.set_types(batch.types)
        flags = (0 if paths else FLAG_NO_PATH) | (0 if payloads else FLAG_NO_JSON) | (FLAG_SKIP_BAD if skip_bad else 0)
        cb, keep = host_cbatch(batch, flags)
        res = CResult()
        rc = self._lib.regk_register_batch(self._h, C.byref(cb), C.byref(res))
        if rc != REGK_OK:
            self._check(rc, res)
        return (res, cb, keep, batch)

    def collect(self, ticket, copy: bool = False) -> HostResult:
        """Wait for a submit()ted batch.  With copy=False the arrays are views of library-owned pinned memory,
        valid until the second following submit()."""
        res = ticket[0]
        rc = self._lib.regk_finish(self._h, C.byref(res))
        if rc != REGK_OK:
            self._check(rc, res)
        n = int(res.n)
        cp = (lambda a: a.copy()) if copy else (lambda a: a)
        out = HostResult(
            n, cp(_as_np(res.path_bytes, int(res.path_total), np.uint8)), cp(_offsets(res, "path_off", n)),
            cp(_as_np(res.json_bytes, int(res.json_total), np.uint8)), cp(_offsets(res, "json_off", n)),
            float(res.kernel_ms), float(res.path_kernel_ms), float(res.json_kernel_ms), int(res.launches),
            float(res.json_len_kernel_ms), int(res.generic_tiles))
        if ticket[1].flags & FLAG_SKIP_BAD:
            out.skipped, out.skipped_bits = self.skipped_records()
        self._lib.regk_release(self._h, C.byref(res))
        return out

    # -- raw access for device-resident callers (bench.py, multi-GPU host layer) --
    def register_raw(self, cbatch: CBatch, cres: Optional[CResult] = None, skip_bad: bool = False) -> CResult:
        """regk_register_batch on a caller-built CBatch.  skip_bad=True adds REGK_SKIP_BAD to its flags; the skipped
        records are then read with skipped_records()."""
        if skip_bad:
            cbatch.flags |= FLAG_SKIP_BAD
        res = cres if cres is not None else CResult()
        rc = self._lib.regk_register_batch(self._h, C.byref(cbatch), C.byref(res))
        self._check(rc, res)
        return res

    def finish(self, cres: CResult) -> CResult:
        self._check(self._lib.regk_finish(self._h, C.byref(cres)), cres)
        return cres

    # -- setupDirectories for the batch finished last (lib/register.js:107-125) --
    def parent_dirs(self, device: bool = False):
        """(parent_len uint32[n], unique_first uint64[n_unique], kernel_ms) for the batch finished last on this
        context: the length of path.dirname(path_i) (always a prefix of path_i) and the record index of the first
        occurrence of every distinct directory, ascending.  device=True returns the raw CParents (device pointers)."""
        out = CParents()
        self._check(self._lib.regk_parent_dirs(self._h, FLAG_OUT_DEVICE if device else 0, C.byref(out)))
        if device:
            return out
        n, nu = int(out.n), int(out.n_unique)
        return (_as_np(out.parent_len, n, np.uint32).copy(), _as_np(out.unique_first, nu, np.uint64).copy(),
                float(out.kernel_ms))

    def mkdirp_dirs(self, device: bool = False):
        """regk_mkdirp_dirs: every directory register()'s setupDirectories must create for the batch finished last
        (each ancestor of each node's directory once, by depth, then by first record) as a DirSet.  device=True
        returns the raw CDirs (device pointers)."""
        out = CDirs()
        self._check(self._lib.regk_mkdirp_dirs(self._h, FLAG_OUT_DEVICE if device else 0, C.byref(out)))
        return out if device else DirSet(out)

    def mkdirp_requests(self, xid_base: int = 1, zk_flags: int = 0, device: bool = False):
        """regk_mkdirp_requests: one CreateRequest (empty data, OPEN_ACL_UNSAFE, zk_flags) per directory of the last
        mkdirp_dirs() call, xid = xid_base + k.  Returns (frame_bytes, frame_off uint64[n_dirs+1], kernel_ms), or the
        raw CFrames with device=True."""
        out = CFrames()
        xid = (int(xid_base) + 2 ** 31) % 2 ** 32 - 2 ** 31
        self._check(self._lib.regk_mkdirp_requests(self._h, xid, int(zk_flags), FLAG_OUT_DEVICE if device else 0,
                                                   C.byref(out)))
        if device:
            return out
        n = int(out.n)
        return (_as_np(out.frame_bytes, int(out.total), np.uint8).copy(), _as_np(out.frame_off, n + 1, np.uint64).copy(),
                float(out.kernel_ms))

    # -- reconcile the batch finished last with a snapshot of the registry --
    def reconcile(self, snapshot, device: bool = False):
        """regk_reconcile: compare the batch finished last with `snapshot` (a batch.Snapshot, host arrays or CUDA
        tensors) and return a Delta, or the raw CDelta (device pointers) with device=True.  Also gathers the requests
        that repair the difference for reconcile_requests()."""
        cin, keep = snapshot.cdecode_in()
        out = CDelta()
        rc = self._lib.regk_reconcile(self._h, C.byref(cin), FLAG_OUT_DEVICE if device else 0, C.byref(out))
        del keep
        self._check(rc)
        return out if device else Delta(out)

    def reconcile_owned(self, snapshot, session: int, zk_flags: int = 1, device: bool = False):
        """regk_reconcile_owned: reconcile() that also weighs each node's Stat - `snapshot` must carry `version` and
        `owner` (Stat.version / Stat.ephemeralOwner per node).  A matched node whose owner is not `session` (zk_flags 1,
        EPHEMERAL) or not 0 (zk_flags 0, persistent) makes its record DELTA_REPLACE.  Returns a Delta with `replace`,
        or the raw CDeltaOwned (device pointers) with device=True."""
        cin, keep = snapshot.cdecode_in()
        st, skeep = snapshot.cnode_stat(int(session), int(zk_flags))
        out = CDeltaOwned()
        rc = self._lib.regk_reconcile_owned(self._h, C.byref(cin), C.byref(st), FLAG_OUT_DEVICE if device else 0,
                                            C.byref(out))
        del keep, skeep
        self._check(rc)
        return out if device else Delta(out.d, out.replace, out.n_replace)

    def reconcile_requests(self, op: int = ZK_CREATE, xid_base: int = 1, zk_flags: int = 1, version: int = -1,
                           group: int = 0, device: bool = False, observed_version: bool = False):
        """regk_reconcile_requests: the create (ZK_CREATE), setData (ZK_SETDATA) or delete (ZK_DELETE) requests of the
        last reconcile(), framed as jute_requests() frames a batch; after reconcile_owned() also the replace multi
        transactions (ZK_REPLACE, group 0 counts as 1), and observed_version=True puts each node's snapshot version
        into its delete / setData / replace frame instead of `version`.  Returns (frame_bytes, frame_off, kernel_ms),
        or the raw CFrames with device=True."""
        xid = (int(xid_base) + 2 ** 31) % 2 ** 32 - 2 ** 31
        flags = (FLAG_OUT_DEVICE if device else 0) | (FLAG_ZK_VERSION_OBSERVED if observed_version else 0)
        o = CJuteOpts(int(op), flags, xid, int(zk_flags), int(version), int(group))
        out = CFrames()
        self._check(self._lib.regk_reconcile_requests(self._h, C.byref(o), C.byref(out)))
        if device:
            return out
        n = int(out.n)
        return (_as_np(out.frame_bytes, int(out.total), np.uint8).copy(), _as_np(out.frame_off, n + 1, np.uint64).copy(),
                float(out.kernel_ms))

    # -- the replies to the getData frames of the batch finished last, as a snapshot --
    def read_replies(self, stream, device: bool = False):
        """regk_read_replies: `stream` (a NumPy uint8 array, or a contiguous CUDA uint8 tensor) holds the bytes read off
        the session after sending the frames of the last jute_requests(op=ZK_GETDATA) call, from the first reply's
        length word on.  Returns a Replies (input of reconcile_owned()), or the raw CReplies (err / node_rec on the
        device) with device=True.  A record whose reply carries an error other than NONODE gets no snapshot node, so a
        reconcile classes it CREATE: do not send the repair while n_error > 0."""
        flags = FLAG_OUT_DEVICE if device else 0
        if hasattr(stream, "data_ptr"):
            import torch
            if not stream.is_cuda or stream.dtype != torch.uint8 or not stream.is_contiguous():
                raise ValueError("a device stream is a contiguous CUDA uint8 tensor")
            keep, ptr, n = stream, stream.data_ptr() or None, stream.numel()
            flags |= FLAG_IN_DEVICE
        else:
            keep = np.ascontiguousarray(stream)
            if keep.dtype != np.uint8 or keep.ndim != 1:
                raise ValueError("a host stream is a one-dimensional uint8 array")
            ptr, n = _np_ptr(keep), keep.size
        out = CReplies()
        rc = self._lib.regk_read_replies(self._h, ptr, n, flags, C.byref(out))
        del keep
        self._check(rc)
        return out if device else Replies(self, out)

    def _d2h(self, ptr, count, dtype):
        out = np.zeros(count, dtype)
        if count:
            self._check(self._lib.regk_memcpy_d2h(self._h, out.ctypes.data_as(C.c_void_p), C.c_void_p(ptr), out.nbytes))
        return out

    # -- multi-GPU reassembly (regk_gather_push over CUDA-IPC mapped peer buffers) --
    def dev_alloc(self, nbytes: int) -> int:
        p = self._lib.regk_dev_alloc(self._h, nbytes)
        if not p:
            raise MemoryError("regk_dev_alloc(%d) failed" % nbytes)
        return p

    def dev_free(self, p: int):
        self._lib.regk_dev_free(self._h, C.c_void_p(p))

    def ipc_export(self, dev_ptr: int) -> bytes:
        buf = C.create_string_buffer(IPC_HANDLE_BYTES)
        self._check(self._lib.regk_ipc_export(self._h, C.c_void_p(dev_ptr), buf))
        return buf.raw

    def ipc_open(self, handle: bytes) -> int:
        out = C.c_void_p()
        self._check(self._lib.regk_ipc_open(self._h, handle, C.byref(out)))
        return out.value

    def ipc_close(self, peer_ptr: int):
        self._lib.regk_ipc_close(self._h, C.c_void_p(peer_ptr))

    def gather_push(self, shard: CResult, plan: CGather):
        self._check(self._lib.regk_gather_push(self._h, C.byref(shard), C.byref(plan)))

    def job_bind(self, job: Optional[CJob]):
        """Bind the multi-GPU job description (regk_job) to the context; None unbinds."""
        self._check(self._lib.regk_job_bind(self._h, C.byref(job) if job is not None else None))

    def memset_dev(self, dev_ptr: int, nbytes: int):
        """Zero device memory allocated with dev_alloc (stream-synchronous helper for non-CUDA hosts)."""
        z = np.zeros(nbytes, np.uint8)
        self._check(self._lib.regk_memcpy_h2d(self._h, C.c_void_p(dev_ptr), z.ctypes.data_as(C.c_void_p), nbytes))

    def host_alloc(self, nbytes: int) -> int:
        p = self._lib.regk_host_alloc(self._h, nbytes)
        if not p:
            raise MemoryError("regk_host_alloc(%d) failed" % nbytes)
        return p

    def host_free(self, p: int):
        self._lib.regk_host_free(self._h, C.c_void_p(p))

    def pinned_array(self, shape, dtype) -> np.ndarray:
        """NumPy array in library-pinned host memory (lives until host_free(arr.ctypes.data))."""
        dt = np.dtype(dtype)
        count = int(np.prod(shape))
        p = self.host_alloc(max(count * dt.itemsize, 1))
        buf = (C.c_uint8 * (count * dt.itemsize)).from_address(p)
        return np.frombuffer(buf, dtype=dt, count=count).reshape(shape)


_default_ctx = {}


def default_context(device: int = 0) -> Context:
    ctx = _default_ctx.get(device)
    if ctx is None:
        ctx = _default_ctx[device] = Context(device)
    return ctx
