"""walk_resolve_util's restatement of regk_walk_resolve's identity and reuse rules on hand-built registries, with the
exact counters each case must give, and the regk_walk_answers layout read from include/regk.h against the ctypes
struct."""
import os
import random

import resolve_util as rv
import walk_resolve_util as wr
import walk_watch_util as ww
from test_resolve_cpu import host, service

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DH, DS = 30, 60
A1 = host(b"redis_host", b"10.0.0.1")
A2 = host(b"redis_host", b"10.0.0.2")
A_LINE = len(b"a.s0.r.\t30\tIN\tA\t10.0.0.1\n")                  # HOST_A section and additional line of /r/s0/a
SA_LINE = len(b"s0.r.\t30\tIN\tA\t10.0.0.1\n")                   # its A line under the service
SRV80 = len(b"_http._tcp.s0.r.\t60\tIN\tSRV\t0 10 80 a.s0.r.\n")
CHILD = SA_LINE + SRV80 + A_LINE                                # /r/s0/a's three child runs


def tree(extra=()):
    zk = ww.WalkZooKeeper()
    for p, d in [(b"/r", b""), (b"/r/s0", service(b"_http", b"_tcp", 80, 60)), (b"/r/s0/a", A1), (b"/r/s0/b", A2)] + list(extra):
        zk.create(p, d, 0, False)
    d = wr.Driver(zk, [b"/r"], random.Random(0))
    d.start()
    return zk, d


def after(zk, d, change):
    """a resolve, then `change`, events and a refresh -> the prediction of the next resolve"""
    d.model.resolved(DH, DS)
    change()
    d.settle()
    return d.model.predict(DH, DS)


def test_first_call_and_changed_ttls_are_full():
    zk, d = tree()
    m = len(d.model.nodes)
    assert d.model.predict(DH, DS) == (1, m, 0)
    d.model.resolved(DH, DS)
    assert d.model.predict(DH, DS) == (0, 0, rv_text(d))
    assert d.model.predict(DH + 1, DS) == (1, m, 0) and d.model.predict(DH, DS + 1) == (1, m, 0)


def rv_text(d):
    r = rv.resolve(d.model.pairs(), DH, DS)
    return sum(len(a) + len(b) for a, b in r["sections"])


def test_instance_deleted_and_added():
    zk, d = tree()
    assert after(zk, d, lambda: zk.delete(b"/r/s0/b")) == (0, 0, 2 * A_LINE + SA_LINE + SRV80)
    zk2, d2 = tree()
    full, fresh, copied = after(zk2, d2, lambda: zk2.create(b"/r/s0/c", host(b"redis_host", b"10.0.0.3"), 0, False))
    assert (full, fresh) == (0, 1) and copied == 2 * (A_LINE + CHILD)


def test_instance_changed_and_identical_rewrite():
    zk, d = tree()
    assert after(zk, d, lambda: zk.set_data(b"/r/s0/b", host(b"redis_host", b"10.0.0.9", 45, [1, 2]))) == (0, 1, A_LINE + CHILD)
    zk, d = tree()
    assert after(zk, d, lambda: zk.set_data(b"/r/s0/b", A2)) == (0, 0, 2 * (A_LINE + CHILD))   # same bytes: kept


def test_service_changed_and_back():
    zk, d = tree()
    assert after(zk, d, lambda: zk.set_data(b"/r/s0", service(b"_http", b"_tcp", 8080, 60))) == (0, 1, 2 * A_LINE)
    zk, d = tree()
    assert after(zk, d, lambda: zk.set_data(b"/r/s0", service(b"_http", b"_tcp", 80, 90))) == (0, 1, 2 * A_LINE)
    zk, d = tree()
    assert after(zk, d, lambda: zk.set_data(b"/r/s0", b"{}")) == (0, 1, 2 * A_LINE)
    assert after(zk, d, lambda: zk.set_data(b"/r/s0", service(b"_http", b"_tcp", 80, 60))) == (0, 1, 2 * A_LINE)


def test_delete_and_recreate_with_the_same_data_is_fresh():
    zk, d = tree()

    def change():
        zk.delete(b"/r/s0/b")
        zk.create(b"/r/s0/b", A2, 0, False)
    full, fresh, copied = after(zk, d, change)
    assert (full, fresh, copied) == (0, 1, A_LINE + CHILD)


def test_types_and_directory_level():
    extra = [(b"/r/s0/o", host(b"ops_host", b"10.0.0.5")), (b"/r/s0/h", host(b"host", b"10.0.0.6")),
             (b"/r/s0/x", host(b"bogus", b"10.0.0.7")), (b"/r/s0/dir", b""), (b"/r/s0/dir/i", host(b"redis_host", b"10.0.0.8"))]
    zk, d = tree(extra)
    d.model.resolved(DH, DS)
    # every node kept its identity: the whole text is copied, the ops_host as a child only, the host as HOST_A only,
    # the bogus type nowhere, the instance under the directory as HOST_A only
    assert d.model.predict(DH, DS) == (0, 0, rv_text(d))
    nodes = d.model.pairs()
    by = {p: n for p, n in zip([n[0] for n in nodes], nodes)}
    assert wr.child_bytes(by[b"/r/s0"], by[b"/r/s0/o"], DH, DS) > 0 and wr.host_a_bytes(by[b"/r/s0/o"], DH, DS) == 0
    assert wr.child_bytes(by[b"/r/s0"], by[b"/r/s0/h"], DH, DS) == 0 and wr.host_a_bytes(by[b"/r/s0/h"], DH, DS) > 0
    assert wr.child_bytes(by[b"/r/s0"], by[b"/r/s0/x"], DH, DS) == 0 and wr.host_a_bytes(by[b"/r/s0/x"], DH, DS) == 0
    assert wr.child_bytes(by[b"/r/s0/dir"], by[b"/r/s0/dir/i"], DH, DS) == 0
    full, fresh, copied = after(zk, d, lambda: zk.set_data(b"/r/s0/o", host(b"ops_host", b"10.0.0.50")))
    assert (full, fresh) == (0, 1) and copied == rv_text(d) - wr.child_bytes(by[b"/r/s0"], d.model.pairs()[
        [n[0] for n in d.model.nodes].index(b"/r/s0/o")], DH, DS)


def test_random_registry_scripts_keep_the_identities_consistent():
    for seed in range(20):
        rng = random.Random(seed)

        def check(d, phase):
            m = d.model
            full, fresh, copied = m.predict(DH, DS)
            assert copied <= rv_text(d) and fresh <= len(m.nodes)
            assert all(i is None or 0 <= i for i in m.ident) and len(m.ident) == len(m.nodes)
            m.resolved(DH, DS)
        wr.script(rng, check, rounds=rng.randrange(2, 6), n_svc=rng.randrange(1, 5), churn=rng.choice([1, 4, 10]))


def test_struct_layout_matches_header(built):
    from registrar_b200 import _native
    with open(os.path.join(ROOT, "include", "regk.h")) as f:
        fields = wr.struct_layout(f.read())
    assert fields == [n for n, _ in _native.CWalkAnswers._fields_]
    import ctypes
    assert _native.CWalkAnswers.answers.offset == 0
    assert _native.CWalkAnswers.n_fresh.offset == ctypes.sizeof(_native.CAnswers)
    assert ctypes.sizeof(_native.CWalkAnswers) == ctypes.sizeof(_native.CAnswers) + 32
