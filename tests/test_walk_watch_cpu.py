"""The watched walk's restatement (walk_watch_util) on its own: random mutation scripts converge on the tree, with
mutations between rounds and while a level is in flight; the named races; the struct layouts against the header."""
import os
import random

import pytest

import events_util as ev
import walk_watch_util as ww

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("seed", range(40))
def test_random_scripts_converge(seed):
    rng = random.Random(seed)
    ww.script(rng, rounds=rng.randrange(2, 9), depth=rng.randrange(1, 5), churn=rng.choice([1, 4, 12]),
              flight=rng.choice([0.0, 0.05, 0.3]), roots=[b"/z"] if seed % 3 else [b"/z", b"/y"])


def _walked(roots=(b"/z",)):
    zk = ww.WalkZooKeeper()
    zk.create(b"/z", b"", 0, False)
    zk.create(b"/z/g", b"g", 0, False)
    zk.create(b"/z/g/p", b"p1", 0, False)
    zk.create(b"/z/g/q", b"q1", 0, False)
    d = ww.Driver(zk, roots, random.Random(0))
    d.start()
    assert d.snapshot_set() == zk.subtree(roots)
    return zk, d


def test_delete_recreate_race():
    """with g's child watch spent, p deleted and recreated between g's getData and getChildren replies: only p's
    NodeDeleted fires, and the parent rule is what makes g pending, so the next refresh walks the new p"""
    d = ww.spent_watch_race()
    assert d.model.counts() == (1, 1)                          # the old p removed, g pending by the parent rule
    g = [n[0] for n in d.model.nodes].index(b"/z/g")
    assert d.model.marks[g] == ww.PENDING
    d.settle()
    assert (b"/z/g/p", b"p2", 0, 0) in d.snapshot_set() and d.snapshot_set() == d.zk.subtree([b"/z"])


def test_delete_recreate_race_needs_the_parent_rule():
    d = ww.spent_watch_race(parent_rule=False)
    assert d.model.counts() == (0, 1)                          # nothing re-lists g
    d.settle()
    assert b"/z/g/p" not in {n[0] for n in d.model.nodes}      # the new p is lost
    assert d.snapshot_set() != d.zk.subtree([b"/z"])


def test_data_changed_between_getdata_and_getchildren():
    zk = ww.WalkZooKeeper()
    zk.create(b"/z", b"", 0, False)
    zk.create(b"/z/a", b"a1", 0, False)
    d = ww.Driver(zk, [b"/z"], random.Random(0))
    d.model.start([b"/z"])
    d.level()                                                  # /z
    xb = d._next_xid(2)
    frames = d.model.requests(xb, True)
    stream = zk.serve(frames, d.SESSION, lambda k: zk.set_data(b"/z/a", b"a2") if k == 0 else None)
    d.model.read(stream)
    assert d.model.nodes[-1][1] == b"a1"                       # the getData reply came before the change
    got = d.model.events(stream, 0, xb, 2)
    assert got["events"][0][4] == 1 and got["n_pending"] == 1
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/z"]) and (b"/z/a", b"a2", 1, 0) in d.snapshot_set()


def test_nonode_on_refresh_getdata():
    zk, d = _walked()
    zk.set_data(b"/z/g/q", b"q2")
    d.feed(zk.take_events(d.SESSION))
    d.model.refresh()
    xb = d._next_xid(2)
    frames = d.model.requests(xb, True)
    zk.delete(b"/z/g/q")                                       # gone before the refresh level is answered
    stream = zk.serve(frames, d.SESSION)
    want = d.model.read(stream)
    assert want["n_missing"] == 1 and b"/z/g/q" not in {n[0] for n in d.model.nodes}
    got = d.model.events(stream, 0, xb, 2)
    assert got["n_unmatched"] == 1                             # q's NodeDeleted: q is no longer a node
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/z"])


def test_deleted_root_stays_gone():
    zk = ww.WalkZooKeeper()
    zk.create(b"/r", b"r", 0, False)
    d = ww.Driver(zk, [b"/r"], random.Random(0))
    d.start()
    zk.delete(b"/r")
    got = d.feed(zk.take_events(d.SESSION))
    assert got["n_removed"] == 1 and got["n_pending"] == 0
    d.settle()
    assert d.model.nodes == []
    zk.create(b"/r", b"back", 0, False)                        # nothing is watching it
    assert zk.take_events(d.SESSION) == b""
    assert d.model.refresh()["n_frontier"] == 0 and d.model.nodes == []


def test_removed_wins_whatever_the_order():
    m = ww.Model()
    m.start([b"/a"])
    m.nodes, m.marks, m.level_off, m.frontier = [(b"/a", b"", 0, 0), (b"/a/b", b"", 0, 0)], [0, 0], [0, 1, 2], []
    for order in ((ev.DELETED, ev.DATA_CHANGED), (ev.DATA_CHANGED, ev.DELETED)):
        m.marks = [0, 0]
        s = b"".join(ev.notification(b"/a/b", t) for t in order)
        got = m.events(s)
        assert [e[4] for e in got["events"]] == [1, 1]         # both see /a/b: the call's own deletes do not hide it
        assert (got["n_pending"], got["n_removed"]) == (1, 1) and m.marks == [1, 3]


def test_struct_layouts_match_header():
    from registrar_b200 import _native
    with open(os.path.join(ROOT, "include", "regk.h")) as f:
        lay = ww.struct_layouts(f.read())
    assert [n for n, _ in _native.CWalkEvents._fields_] == lay["regk_walk_events_out"]
    assert [n for n, _ in _native.CWalkRefresh._fields_] == lay["regk_walk_refresh_out"]
    assert "regk_walk_events" in _native.EXPORTS and "regk_walk_refresh" in _native.EXPORTS
