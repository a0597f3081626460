"""A watched walk across a reconnect, restated (walk_setwatches_util) on its own: the SetWatches frames of the
README's authcache tree pinned byte for byte, a deleted node firing NodeDeleted twice, random drop scripts converging
on the tree with the pending-and-removed set after every resume checked exactly, and the struct layout against the
header."""
import os
import random
import struct

import pytest

import events_util as ev
import setwatches_util as sw
import walk_setwatches_util as ws
from test_resolve_cpu import AC1, AC2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATHS = [b"/us/joyent", b"/us/joyent/emy-10", b"/us/joyent/emy-10/authcache", b"/us/joyent/emy-10/authcache/" + AC1,
         b"/us/joyent/emy-10/authcache/" + AC2]
REL = 0x100000006                       # six creates, each one zxid past 0x100000000; every reply carries the last


def _entries(paths):
    return b"".join(struct.pack(">i", len(p)) + p for p in paths)


def test_readme_frames_pinned():
    """worked by hand: one frame, xid -8, op 101, relativeZxid, D = the five nodes in walk order, E empty, C = D"""
    zk, d = ws.readme_walked()
    assert [n[0] for n in d.model.nodes] == PATHS and d.model.mark == REL
    want = d.model.setwatches()
    body = (b"\xff\xff\xff\xf8" + b"\x00\x00\x00\x65" + b"\x00\x00\x00\x01\x00\x00\x00\x06" +
            b"\x00\x00\x00\x05" + _entries(PATHS) + b"\x00\x00\x00\x00" + b"\x00\x00\x00\x05" + _entries(PATHS))
    assert len(body) == 28 + 2 * sum(4 + len(p) for p in PATHS) == 432
    assert want["frames"] == struct.pack(">i", len(body)) + body and want["frame_off"] == [0, 436]
    assert (want["n_listed"], want["n_repend"], want["n_frontier"], want["relative_zxid"]) == (5, 0, 0, REL)


def test_readme_frames_split_at_the_minimum():
    """max_frame = 32 + 2 (4 + 64) = 168: B = 68, so entry j goes into frame s_j // 68, s_j the prefix of the entry
    sizes 14, 21, 31, 68, 68 (D), then the same again (C)"""
    zk, d = ws.readme_walked()
    lmax = len(PATHS[3])
    assert lmax == 64
    want = d.model.setwatches(32 + 2 * (4 + lmax))
    sizes = [4 + len(p) for p in PATHS * 2]
    s = [sum(sizes[:j]) for j in range(10)]
    assert s == [0, 14, 35, 66, 134, 202, 216, 237, 268, 336]
    assert [x // 68 for x in s] == [0, 0, 0, 0, 1, 2, 3, 3, 3, 4]
    frames = sw.parse(want["frames"])
    assert [(len(D), len(E), len(C)) for _, D, E, C in frames] == [(4, 0, 0), (1, 0, 0), (0, 0, 1), (0, 0, 3), (0, 0, 1)]
    assert all(rel == REL for rel, _, _, _ in frames)
    assert all(b - a < 32 + 2 * (4 + lmax) for a, b in zip(want["frame_off"], want["frame_off"][1:]))


def test_deleted_node_fires_nodedeleted_twice():
    """an instance deleted while the connection is down: listed in D and in C, it fires NodeDeleted twice; the node is
    removed once and its parent, whose pzxid moved, is pending"""
    zk, d = ws.readme_walked()
    zk.drop_connection(d.SESSION)
    zk.delete(PATHS[4])
    want = d.model.setwatches()
    stream = zk.serve_setwatches(want["frames"], d.SESSION)
    got = d.model.events(stream)
    assert [(e[1], e[4]) for e in got["events"]] == [(ev.DELETED, 4), (ev.CHILDREN_CHANGED, 2), (ev.DELETED, 4)]
    assert (got["n_pending"], got["n_removed"], got["n_replies"]) == (1, 1, 1)
    d.levels()
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/us/joyent"])


def test_changed_while_down_is_exactly_what_is_pending():
    """a setData, a create and a delete while down: exactly the nodes they touched are pending or removed"""
    zk, d = ws.readme_walked()
    zk.drop_connection(d.SESSION)
    zk.set_data(PATHS[2], b"{}")
    zk.create(PATHS[1] + b"/other", b"", 0, False)
    want = ws.check_resume(d)
    assert want["n_listed"] == 5 and want["n_repend"] == 0
    assert [j for j, mk in enumerate(d.model.marks) if mk] == [1, 2]
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/us/joyent"])


def test_errors_and_in_flight_levels_are_repended_or_left_alone():
    """a getChildren error leaves the node unarmed (re-pended); a level in flight is left for the caller to frame
    again, and its nodes are not snapshot nodes yet"""
    zk, d = ws.readme_walked()
    zk.fail[(8, PATHS[2])] = -102                              # NOAUTH on authcache's listing
    zk.set_data(PATHS[2], b"x")
    d.feed(zk.take_events(d.SESSION))
    d.refresh()
    assert d.model.armed == [True, True, False, True, True]
    want = d.model.setwatches()
    assert (want["n_listed"], want["n_repend"]) == (4, 1) and d.model.marks[2] == ws.PENDING
    del zk.fail[(8, PATHS[2])]
    zk.drop_connection(d.SESSION)
    d.feed(zk.serve_setwatches(want["frames"], d.SESSION))
    d.settle()
    assert d.snapshot_set() == zk.subtree([b"/us/joyent"])


def test_refused_calls_change_nothing():
    zk, d = ws.readme_walked()
    marks, gate = list(d.model.marks), d.model.gate
    for mf in (32 + 2 * 68 - 1, 2 ** 31):
        with pytest.raises(ws.Refused):
            d.model.setwatches(mf)
    assert d.model.marks == marks and d.model.gate == gate
    d.model.setwatches(32 + 2 * 68)
    assert d.model.gate


def test_gate():
    """-8 is refused before a SetWatches framing and accepted after it; a -8 frame with a body or an err never is"""
    zk, d = ws.readme_walked()
    with pytest.raises(ev.Refused):
        d.model.events(sw.reply(5))
    d.model.setwatches()
    assert d.model.events(sw.reply(REL + 9))["n_replies"] == 1 and d.model.mark == REL + 9
    for bad, code in ((sw.reply(5, body=b"x"), sw.SW_BODY), (sw.reply(5, err=-4), sw.SW_ERR)):
        with pytest.raises(ev.Refused) as e:
            d.model.events(bad)
        assert e.value.code == code


@pytest.mark.parametrize("seed", range(40))
def test_random_drop_scripts_converge(seed):
    rng = random.Random(seed)
    ws.script(rng, drops=rng.randrange(1, 5), depth=rng.randrange(1, 5), churn=rng.choice([1, 4, 10]),
              roots=[b"/z"] if seed % 3 else [b"/z", b"/y"], max_frame=rng.choice([0, 0, 300]))


def test_struct_layout_matches_header():
    from registrar_b200 import _native
    with open(os.path.join(ROOT, "include", "regk.h")) as f:
        fields = ws.struct_fields(f.read(), "regk_walk_setwatches_out")
    assert [n for n, _ in _native.CWalkSetWatches._fields_] == fields
    assert "regk_walk_setwatches" in _native.EXPORTS
