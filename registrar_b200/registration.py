"""register() / unregister() — host-side mirror of the reference's lib/register.js.

Same names, argument shape, callback discipline and error behaviour as the reference
(/root/reference/lib/register.js), with the per-record compute (rows A1–A4 of SURVEY.md §8: domain ->
znode path, host-record payload bytes) done on the GPU through the C-ABI (libregk.so) instead of V8:

    register(opts, cb)      lib/register.js:174-251     cb(err) | cb(None, znodes)
    unregister(opts, cb)    lib/register.js:254-295
    domain_to_path(domain)  lib/register.js:34-39       (module-private there; exported here for tools)
    register_batch(...)     new: N records in one call (the batch dimension of BASELINE.json)

What crosses the `opts['zk']` seam (duck-typed client: unlink, mkdirp, create, put — register.js:62,87,116,159):
the reference hands zk.create() a JS object that zkplus serialises; this module hands it the payload BYTES
the GPU produced (exactly what zkplus would have put on the wire), with
``{'flags': ['ephemeral_plus'], 'serialized': True}``.  zk.put() for the service record receives the dict,
as in the reference (register.js:58-62) — that row is not on the GPU path yet (SURVEY.md §8f-1).

Argument errors raise AssertionError synchronously (assert-plus behaviour, register.js:175-201); runtime
failures go to the callback.  There is no CPU implementation of the path here: without libregk.so and a
CUDA device the call raises.
"""
from __future__ import annotations

import os
import socket
import threading
from typing import Callable, Iterable, List, Optional

from . import _native
from .batch import RecordBatch

WAIT_MS = 1000          # "Be nice to watchers and wait for them to catch up" (register.js:232-235)


# --------------------------------------------------------------------------- assert-plus look-alikes
def _fail(name, typ):
    raise AssertionError("%s (%s) is required" % (name, typ))


def _a_object(v, name):
    if not isinstance(v, dict) and not (hasattr(v, "__dict__") and not callable(v)):
        _fail(name, "object")


def _a_string(v, name):
    if not isinstance(v, str):
        _fail(name, "string")


def _a_number(v, name):
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        _fail(name, "number")


def _a_func(v, name):
    if not callable(v):
        _fail(name, "func")


def _opt(check):
    return lambda v, name: None if v is None else check(v, name)


def _a_array_of(check, typ):
    def f(v, name):
        if not isinstance(v, (list, tuple)):
            _fail(name, "[%s]" % typ)
        for x in v:
            try:
                check(x, name)
            except AssertionError:
                _fail(name, "[%s]" % typ)
    return f


_a_array_of_string = _a_array_of(_a_string, "string")
_a_array_of_number = _a_array_of(_a_number, "number")


def _get(o, k, default=None):
    return o.get(k, default) if isinstance(o, dict) else getattr(o, k, default)


def once(fn: Callable) -> Callable:
    state = {"done": False, "value": None}

    def wrapper(*a, **kw):
        if state["done"]:
            return state["value"]
        state["done"] = True
        state["value"] = fn(*a, **kw)
        return state["value"]
    return wrapper


# ----------------------------------------------------------------------------- vasync look-alikes
def for_each_parallel(func, inputs, cb):
    inputs = list(inputs)
    if not inputs:
        cb(None)
        return
    st = {"pending": len(inputs), "err": None}

    def mk():
        def done(err=None, *_):
            if err is not None and st["err"] is None:
                st["err"] = err
            st["pending"] -= 1
            if st["pending"] == 0:
                cb(st["err"])
        return once(done)
    for x in inputs:
        func(x, mk())


def for_each_pipeline(func, inputs, cb):
    it = iter(list(inputs))

    def nxt(err=None, *_):
        if err is not None:
            cb(err)
            return
        try:
            x = next(it)
        except StopIteration:
            cb(None)
            return
        func(x, nxt)
    nxt()


def pipeline(funcs, arg, cb):
    it = iter(funcs)

    def nxt(err=None, *_):
        if err is not None:
            cb(err)
            return
        try:
            f = next(it)
        except StopIteration:
            cb(None)
            return
        f(arg, nxt)
    nxt()


def _default_timer(ms, fn):
    t = threading.Timer(ms / 1000.0, fn)
    t.daemon = True
    t.start()
    return t


# ------------------------------------------------------------------------------------- GPU helpers
def _ctx(opts=None) -> _native.Context:
    c = _get(opts, "_regk", None) if opts is not None else None
    return c if c is not None else _native.default_context(int(os.environ.get("REGK_DEVICE", "0")))


def _first_address() -> str:
    # lib/register.js:22-31 address(): first non-internal interface.  Resolved on the host, once.
    s = socket.socket(socket.AF_INET, socket.SOCK_DGRAM)
    try:
        s.connect(("10.255.255.255", 1))
        return s.getsockname()[0]
    except OSError:
        raise RuntimeError("no adminIp given and no non-internal interface address found")
    finally:
        s.close()


def domain_to_path(domain, ctx: Optional[_native.Context] = None) -> str:
    """'1.moray.us-east.joyent.com' -> '/com/joyent/us-east/moray/1' (register.js:34-39), on the GPU."""
    _a_string(domain, "domain")
    rec = {"domain": domain, "hostname": "", "type": "host", "address": "0"}
    res = (ctx or _ctx()).register_batch(RecordBatch.from_records([rec], alias=True), payloads=False)
    return res.path(0).decode("utf-8")


def register_batch(records: Iterable[dict], cb: Optional[Callable] = None, ctx: Optional[_native.Context] = None,
                   alias: bool = False, skip_bad: bool = False):
    """N host records -> (paths, payloads) in one GPU call.

    records: dicts {domain, hostname, type, address (adminIp), ttl?, ports?}.  Returns the HostResult
    (path(i) / json(i) accessors, packed byte streams + offsets) and, when cb is given, also calls
    cb(None, result) / cb(err).  skip_bad=True: a record outside the supported input domain no longer refuses
    the whole batch; it comes back with an empty path and payload and is listed in result.skipped (record
    indices) / result.skipped_bits, for the caller to route to another implementation."""
    try:
        res = (ctx or _ctx()).register_batch(RecordBatch.from_records(records, alias=alias), skip_bad=skip_bad)
    except Exception as e:  # noqa: BLE001
        if cb is None:
            raise
        cb(e)
        return None
    if cb is not None:
        cb(None, res)
    return res


def _node_dirname(p: str) -> str:
    """node (>= 6) posix path.dirname, as used at register.js:118 (control-plane string op on a handful of
    znode names per call; the batched variant is SURVEY.md §8f-2)."""
    if not p:
        return "."
    has_root = p[0] == "/"
    i = len(p) - 1
    while i >= 1 and p[i] == "/":
        i -= 1
    j = p.rfind("/", 1, i + 1)
    if j == -1:
        return "/" if has_root else "."
    if has_root and j == 1:
        return "//"
    return p[:j]


# ------------------------------------------------------------------------------------ pipeline steps
class Serialized(bytes):
    """A znode payload already serialised by the GPU path: the client sends these bytes as they are instead of
    JSON.stringify-ing an object (zk.create gets the same through its `serialized` option)."""


def service_payloads(services: Iterable[dict], ctx: Optional[_native.Context] = None):
    """N `registration.service` objects -> the payloads of their service records, one GPU call (SURVEY §8f-1)."""
    from .batch import ServiceBatch
    return (ctx or _ctx()).service_records(ServiceBatch.from_services(services))


def _register_service(opts, cb):
    # lib/register.js:45-75.  The record {type:'service', service: registration.service} is serialised on the
    # GPU (regk_service_records); members outside srvce/proto/port/ttl are not representable there and raise.
    if not _get(opts["registration"], "service"):
        cb()
        return
    cb = once(cb)
    try:
        obj = Serialized(service_payloads([_get(opts["registration"], "service")], _ctx(opts)).json(0))
    except Exception as e:  # noqa: BLE001
        cb(e)
        return

    def done(err=None, *_):
        if err:
            cb(err)
        else:
            if opts["path"] not in opts["nodes"]:
                opts["nodes"].append(opts["path"])
            cb()
    opts["zk"].put(opts["path"], obj, done)


def _cleanup_previous_entries(opts, cb):
    # lib/register.js:78-105
    def unlink(n, _cb):
        def done(err=None, *_):
            if err and getattr(err, "name", None) != "NO_NODE":
                _cb(err)
            else:
                _cb()
        opts["zk"].unlink(n, done)
    for_each_parallel(unlink, opts["nodes"], once(cb))


def _setup_directories(opts, cb):
    # lib/register.js:108-129: mkdirp(path.dirname(n)) for every node
    dirs = [_node_dirname(n) for n in opts["nodes"]]
    for_each_parallel(lambda d, _cb: opts["zk"].mkdirp(d, _cb), dirs, once(cb))


def _register_entries(opts, cb):
    # lib/register.js:132-171.  The payload bytes were produced on the GPU (A3/A4); every node of one
    # registration carries the same record.
    payload = opts["payload"]

    def create(n, _cb):
        opts["zk"].create(n, payload, {"flags": ["ephemeral_plus"], "serialized": True}, once(_cb))
    for_each_parallel(create, opts["nodes"], once(cb))


# --------------------------------------------------------------------------------------- public API
def register(opts, cb):
    """lib/register.js:174-251."""
    _a_object(opts, "options")
    _a_object(_get(opts, "log"), "options.log")
    _opt(_a_string)(_get(opts, "adminIp"), "options.adminIp")
    aliases = _get(opts, "aliases")
    if aliases is not None and not isinstance(aliases, (list, tuple, dict)):
        _fail("options.aliases", "object")
    _a_string(_get(opts, "domain"), "options.domain")
    reg = _get(opts, "registration")
    _a_object(reg, "options.registration")
    _a_string(_get(reg, "type"), "options.registration.type")
    _opt(_a_number)(_get(reg, "ttl"), "options.registration.ttl")
    _opt(_a_array_of_number)(_get(reg, "ports"), "options.registration.ports")
    svc = _get(reg, "service")
    if svc is not None:
        _a_object(svc, "options.registration.service")
    if svc:
        _a_string(_get(svc, "type"), "options.registration.service.type")
        assert _get(svc, "type") == "service"
        s2 = _get(svc, "service")
        _a_object(s2, "options.registration.service.service")
        _a_string(_get(s2, "srvce"), "options.registration.service.service.srvce")
        _a_string(_get(s2, "proto"), "options.registration.service.service.proto")
        _opt(_a_number)(_get(s2, "ttl"), "options.registration.service.service.ttl")
        if _get(s2, "ttl") is None:
            s2["ttl"] = 60                                   # register.js:197 (mutates the caller's object)
        _a_number(_get(s2, "port"), "options.registration.service.service.port")
    _a_object(_get(opts, "zk"), "options.zk")
    _a_func(cb, "callback")

    cb = once(cb)
    ctx = _ctx(opts)
    hostname = _get(opts, "_hostname") or socket.gethostname()           # os.hostname(), register.js:222
    alias_list = list(aliases or [])

    # registration.ports, else [service.service.port] (register.js:146-150); [] is truthy in JS
    ports = _get(reg, "ports")
    if ports is None and svc:
        ports = [_get(_get(svc, "service"), "port")]
    address = _get(opts, "adminIp") or _first_address()                  # register.js:143
    ttl = _get(reg, "ttl")
    for v in ([ttl] if ttl is not None else []) + list(ports or []):
        if isinstance(v, float) and not v.is_integer():
            raise AssertionError("non-integer numbers are outside the GPU path's input domain: %r" % (v,))

    try:
        host = ctx.register_batch(RecordBatch.from_records([{
            "domain": opts["domain"] if isinstance(opts, dict) else opts.domain, "hostname": hostname,
            "type": _get(reg, "type"), "address": address, "ttl": None if ttl is None else int(ttl),
            "ports": None if ports is None else [int(x) for x in ports]}]))
        names = [_get(opts, "domain")] + alias_list                      # p itself + the alias nodes: A1, un-normalised
        for a in alias_list:
            _a_string(a, "domain")
        al = ctx.register_batch(RecordBatch.from_records(
            [{"domain": d, "hostname": "", "type": _get(reg, "type"), "address": address} for d in names], alias=True),
            payloads=False)
    except _native.RegkError as e:
        cb(e)
        return
    p = al.path(0).decode("utf-8")
    cookie = {
        "adminIp": _get(opts, "adminIp"), "domain": _get(opts, "domain"), "log": _get(opts, "log"),
        "nodes": [host.path(0).decode("utf-8")] + [al.path(i + 1).decode("utf-8") for i in range(len(alias_list))],
        "path": p, "registration": reg, "zk": _get(opts, "zk"), "payload": host.json(0),
    }
    timer = _get(opts, "_setTimeout") or _default_timer
    wait_ms = _get(opts, "_waitMs", WAIT_MS)

    def wait(_, _cb):
        timer(wait_ms, once(_cb))

    def done(err=None):
        if err:
            cb(err)
        else:
            cb(None, cookie["nodes"])
    pipeline([_cleanup_previous_entries, wait, _setup_directories, _register_entries, _register_service], cookie, done)


def unregister(opts, cb):
    """lib/register.js:254-295 — including its quirk: the per-node success path calls the OUTER callback
    (register.js:281), so the pipeline never advances past the first znode and cb fires once."""
    _a_object(opts, "options")
    _a_object(_get(opts, "log"), "options.log")
    _a_object(_get(opts, "zk"), "options.zk")
    _a_array_of_string(_get(opts, "znodes"), "options.znodes")
    _a_func(cb, "callback")
    cb = once(cb)
    zk = _get(opts, "zk")

    def cleanup(n, _cb):
        _cb = once(_cb)

        def done(err=None, *_):
            if err:
                _cb(err)
            else:
                cb()
        zk.unlink(n, done)
    for_each_pipeline(cleanup, _get(opts, "znodes"), lambda err=None: cb(err) if err else cb())
