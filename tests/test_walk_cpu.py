"""The registry walk without a GPU: the restatement in walk_util walks the reference README's authcache tree (two
levels of directories, the service record, its two redis_host instances) through frames and replies built and parsed
byte for byte; the root rule; the races and errors its reader sees; the C-ABI struct layout of regk_walk."""
import ctypes as C
import os
import random
import subprocess
import tempfile

import pytest

import replies_util as ru
import walk_util as wu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AUTH = b"/us/joyent/emy-10/authcache"


def frames(paths, xid_base):
    """the two-section buffer regk_walk_requests frames, restated"""
    return ru.getdata_frames(paths, xid_base) + wu.cu.getchildren_frames(paths, wu.wrap(xid_base + len(paths)))


def walk(tree, roots, xid_base=1, **knobs):
    """the restatement's level loop: (nodes, level_off, per-level reads)"""
    nodes, off, reads, frontier, xid = [], [0], [], list(roots), xid_base
    while frontier:
        fb = frames(frontier, xid)
        assert wu.parse_requests(fb, xid) == frontier
        r = wu.read_level(wu.answer(tree, fb, xid, **knobs), frontier, xid)
        reads.append(r)
        nodes += r["nodes"]
        off.append(len(nodes))
        xid, frontier = wu.wrap(xid + 2 * len(frontier)), r["frontier"]
    return nodes, off, reads


def test_readme_tree():
    t = wu.readme_tree()
    nodes, off, reads = walk(t, [b"/us/joyent"])
    assert [p for p, *_ in nodes] == [b"/us/joyent", b"/us/joyent/emy-10", AUTH, AUTH + b"/" + b"a2674d3b-a9c4-46bc-a835-b6ce21d522c2",
                                      AUTH + b"/" + b"a4ae094d-da07-4911-94f9-c982dc88f3cc"]
    assert off == [0, 1, 2, 3, 5] and (nodes, off) == wu.bfs(t, [b"/us/joyent"])
    assert nodes[2][1].startswith(b'{"type":"service"') and nodes[2][2] == 2
    assert all(v == 1 and o == 0x100000001 and b'"redis_host"' in d for _, d, v, o in nodes[3:])
    assert [r["n_children"] for r in reads] == [1, 1, 2, 0]
    assert reads[-1]["n_found"] == 2 and reads[-1]["n_listed"] == 2 and reads[-1]["frontier"] == []


def test_readme_frames_by_hand():
    """frame 0 and frame 1 of the one-root framing, worked out from zookeeper.jute"""
    fb = frames([AUTH], 7)
    p = len(AUTH)
    assert fb[:4 + 13 + p] == (13 + p).to_bytes(4, "big") + (7).to_bytes(4, "big") + (4).to_bytes(4, "big") + \
        p.to_bytes(4, "big") + AUTH + b"\x00"
    assert fb[17 + p:] == (13 + p).to_bytes(4, "big") + (8).to_bytes(4, "big") + (8).to_bytes(4, "big") + \
        p.to_bytes(4, "big") + AUTH + b"\x00"


def test_races_errors_and_noise():
    rng = random.Random(3)
    t = wu.readme_tree()

    def between(tree, paths):            # the service vanishes between its getData and its getChildren
        if AUTH in paths:
            tree.remove(AUTH)
    nodes, off, reads = walk(t, [b"/us"], between=between)
    assert [p for p, *_ in nodes][-1] == AUTH and reads[-1]["n_list_missing"] == 1 and off[-1] == 4
    t = wu.readme_tree()
    nodes, _, reads = walk(t, [b"/us"], rng=rng, noise=5, shuffle=True, null=True, gd_errors={0: -4})
    # every level's node 0 fails its getData, yet its listing still leads the walk down to the instances
    assert [r["n_error"] for r in reads] == [1] * 5 and len(nodes) == 1 and nodes[0][0].startswith(AUTH + b"/")
    assert sum(r["n_skipped"] for r in reads) <= 5 * len(reads)


@pytest.mark.parametrize("roots,want", [
    ([b"/a"], None), ([b"/a", b"/b", b"/ab"], None),
    ([b"/a", b"/"], (1, "/")), ([b"a"], (0, "rejects")), ([b"/a/"], (0, "rejects")), ([b""], (0, "rejects")),
    ([b"/a//b"], (0, "rejects")), ([b"/a\x01"], (0, "rejects")), ([b"/a", b"/b", b"/a"], (2, "equals")),
    ([b"/a/b", b"/a"], (0, "under")), ([b"/a", b"/a/b/c"], (1, "under")), ([b"/x", b"/ab", b"/a"], None)])
def test_root_rule(roots, want):
    assert wu.root_error(roots) == want


def test_struct_layout_matches_header(built):
    from registrar_b200 import _native
    W = _native.CWalk
    names = [f[0] for f in W._fields_]
    src = "#include <stddef.h>\n#include <stdio.h>\n#include \"regk.h\"\nint main(void) {\n"
    src += 'printf("%zu\\n", sizeof(regk_walk));\n'
    src += "".join('printf("%%zu\\n", offsetof(regk_walk, %s));\n' % n for n in names)
    src += "return 0; }\n"
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "t.c"), "w") as f:
            f.write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"), os.path.join(d, "t.c")])
        got = [int(x) for x in subprocess.check_output([os.path.join(d, "t")]).split()]
    assert got == [C.sizeof(W)] + [getattr(W, n).offset for n in names]
    assert {"regk_walk_start", "regk_walk_requests", "regk_read_walk"} <= set(_native.EXPORTS)
