"""Independent restatement of the mkdirp set of a batch (regk_mkdirp_dirs / regk_mkdirp_requests), for the tests.

setupDirectories (lib/register.js:107-129) calls zk.mkdirp(path.dirname(n)) for every node; mkdirp creates the
directory and every ancestor.  Built on pyoracle.node_dirname (pinned by the reference's own mkdirp arguments) and
pyoracle.jute_create_request (the published CreateRequest layout).
"""
from oracle import pyoracle


def dir_of(path: bytes) -> bytes:
    return pyoracle.node_dirname(path.decode("latin-1")).encode("latin-1")


def zk_rejects(d: bytes) -> bool:
    """ZooKeeper's path check on a directory this library can produce (bytes >= 0x80 and '.' / '..' components are
    outside its domain fence): no leading '/', an empty component, a trailing '/', or a byte in 0x00-0x1F / 0x7F."""
    if d in (b"", b"/"):
        return False
    return (not d.startswith(b"/") or d.endswith(b"/") or b"//" in d or
            any(c < 0x20 or c == 0x7F for c in d))


def components(d: bytes):
    """None when ZooKeeper rejects d, else the number of components ("/" and "" have none)."""
    if zk_rejects(d):
        return None
    return 0 if d in (b"", b"/") else d.count(b"/")


def ancestors(d: bytes):
    """every prefix of a valid directory that ends at a component boundary, shortest first, d itself last"""
    if components(d) in (None, 0):
        return []
    return [d[:k] for k in range(1, len(d)) if d[k:k + 1] == b"/"] + [d]


def mkdirp_set(paths):
    """(dirs, first, invalid): the directories in creation order (depth, then first record whose directory has them as a
    prefix), that first record of each, and the first record of every distinct rejected directory, ascending."""
    first, invalid, seen_bad = {}, [], set()
    for i, p in enumerate(paths):
        d = dir_of(p)
        if zk_rejects(d):
            if d not in seen_bad:
                seen_bad.add(d)
                invalid.append(i)
            continue
        for a in ancestors(d):
            first.setdefault(a, i)
    dirs = sorted(first, key=lambda a: (a.count(b"/"), first[a]))
    return dirs, [first[a] for a in dirs], invalid


def mkdirp_frames(dirs, xid_base: int, zk_flags: int) -> bytes:
    wrap = lambda x: (x + 2 ** 31) % 2 ** 32 - 2 ** 31
    return b"".join(pyoracle.jute_create_request(d, b"", wrap(xid_base + k), zk_flags) for k, d in enumerate(dirs))
