"""Stream generators and mutators for the reply-stream reader fuzz test (test_reader_fuzz.py): frames split and
interleaved, decoy frames hidden in notification paths, pads that place a frame head at a chosen byte, the candidate
positions of a stream under a reader's plausibility restatement, and byte-level mutations.  Every stream is plain bytes;
nothing here touches a GPU."""
import struct

import numpy as np

import events_util as eu
import replies_util as ru

SPAN = 2048                 # stream bytes per candidate CTA
SUPER_BYTES = 64 * SPAN     # one super-tile of candidate CTAs (64 tiles)


def be32(b, k):
    return struct.unpack_from(">i", b, k)[0]


def split(b):
    """back-to-back frames -> [frame bytes]"""
    out, k = [], 0
    while k < len(b):
        ln = be32(b, k)
        out.append(b[k:k + 4 + ln])
        k += 4 + ln
    return out


def notification_of_len(total, typ=eu.DATA_CHANGED, fill=b"\xa5"):
    """a notification frame of exactly `total` (>= 32) bytes, its path `fill` repeated"""
    assert total >= 32
    return eu.notification((fill * (total - 32))[:total - 32], typ)


def decoy(payload, total=None, typ=eu.DATA_CHANGED):
    """a notification whose path is `payload` (copies of well-formed frames: false candidates inside a true frame).
    Its zxid is 0, not -1: past 1 MiB the length word's low half and the xid -1 after it would make byte 2 a head."""
    f = eu.notification(payload, typ, zxid=0)
    return f if total is None else notification_of_len(total) if total != len(f) else f


def pad_to(at, target):
    """a notification that, placed at byte `at`, ends exactly at `target` (so the next frame's head sits there);
    target - at >= 32"""
    return notification_of_len(target - at)


def interleave(frames, rng, extras):
    """frames with each of `extras` inserted before a random frame (or after the last)"""
    out = list(frames)
    for x in extras:
        out.insert(rng.randrange(len(out) + 1), x)
    return out


def noise(rng, paths, k):
    """k pings and notifications for paths of the batch (and a few other paths)"""
    out = []
    for _ in range(k):
        c = rng.randrange(4)
        if c == 0:
            out.append(ru.ping())
        else:
            p = rng.choice(paths) if paths and c < 3 else b"/other/%d" % rng.randrange(100)
            out.append(eu.notification(p, rng.choice([1, 2, 3, 4]), zxid=rng.getrandbits(40)))
    return out


def cands(head, b, start=0):
    """positions >= start whose frame head passes `head(b, pos)` (a reader's plausibility restatement): every test
    refuses a length below 16 or past the stream, so only those positions are asked"""
    a = np.frombuffer(bytes(b), np.uint8)
    n = a.size
    if n - start < 4:
        return []
    w = a.astype(np.int64)
    L = (w[:-3] << 24 | w[1:-2] << 16 | w[2:-1] << 8 | w[3:]).astype(np.uint32).view(np.int32).astype(np.int64)
    pos = np.arange(L.size)
    ok = (L >= 16) & (L + 4 <= n - pos) & (pos >= start)
    return [int(p) for p in np.nonzero(ok)[0] if head(b, int(p)) == 0]


# ---- mutators: (stream, frame starts, rng) -> (stream, a short description) ----

def _starts(b, start=0):
    out, k = [], start
    while k + 4 <= len(b):
        out.append(k)
        ln = be32(b, k)
        if ln < 16:
            break
        k += 4 + ln
    return out


def m_header_byte(b, rng, start):
    s = _starts(b, start)
    if not s:
        return b, "none"
    f = rng.choice(s)
    o = rng.choice([0, 1, 2, 3, 4, 5, 6, 7, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31])
    if f + o >= len(b):
        return b, "none"
    x = bytearray(b)
    x[f + o] = rng.choice([x[f + o] ^ (1 << rng.randrange(8)), rng.randrange(256), 0, 0xFF])
    return bytes(x), "header byte %d of the frame at %d" % (o, f)


def m_len_word(b, rng, start):
    s = _starts(b, start)
    if not s:
        return b, "none"
    f = rng.choice(s)
    if f + 4 > len(b):
        return b, "none"
    d = rng.choice([-16, -1, 1, 16])
    x = bytearray(b)
    x[f:f + 4] = struct.pack(">i", (be32(b, f) + d + 2 ** 31) % 2 ** 32 - 2 ** 31)
    return bytes(x), "len %+d at %d" % (d, f)


def m_delete(b, rng, start):
    if len(b) <= start + 1:
        return b, "none"
    i = rng.randrange(start, len(b))
    j = min(len(b), i + rng.choice([1, 2, 4, 8, 16, 37]))
    return b[:i] + b[j:], "delete %d..%d" % (i, j)


def m_insert(b, rng, start):
    i = rng.randrange(start, len(b) + 1)
    ins = rng.choice([bytes([rng.randrange(256)]), b"\x00" * 4, ru.ping(), ru.ping()[:rng.randrange(1, 20)]])
    return b[:i] + ins + b[i:], "insert %d bytes at %d" % (len(ins), i)


def m_truncate(b, rng, start):
    if len(b) <= start:
        return b, "none"
    i = rng.randrange(start, len(b))
    return b[:i], "truncate at %d" % i


def m_splice(b, rng, start):
    fr = split_from(b, start)
    if len(fr) < 2:
        return b, "none"
    i, j = rng.randrange(len(fr)), rng.randrange(len(fr))
    a, c = fr[i], fr[j]
    cut = rng.randrange(1, max(2, min(len(a), len(c))))
    fr[i] = a[:cut] + c[cut:]
    return b[:start] + b"".join(fr), "splice frame %d into %d at %d" % (j, i, cut)


def split_from(b, start):
    """the frames from `start` while their lengths chain (the rest as one piece)"""
    out, k = [], start
    while k < len(b):
        ln = be32(b, k) if k + 4 <= len(b) else -1
        if ln < 16 or k + 4 + ln > len(b):
            out.append(b[k:])
            break
        out.append(b[k:k + 4 + ln])
        k += 4 + ln
    return out


MUTATORS = [m_header_byte, m_len_word, m_delete, m_insert, m_truncate, m_splice]


def mutate(b, rng, k, start=0):
    """0 .. k mutations of b from `start` on -> (stream, [descriptions])"""
    what = []
    for _ in range(rng.randrange(k + 1)):
        b, d = rng.choice(MUTATORS)(b, rng, start)
        what.append(d)
    return b, what


def long_front(start, rng):
    """`start` bytes before the stream a reader reads from `start`.  From 32 bytes on they form a plausible chain from
    byte 0 that leads past `start`: pings, then a notification head whose length claims 7 bytes beyond `start` (so a
    reader that starts at 0 lands inside the real stream).  From 8 to 31 bytes they hold only a length word and xid
    -1 claiming the same end (or byte 20, if later): plausible to the readers that skip an xid -1 frame whatever its
    body, while the events reader's test of the notification body reads the real stream.  Below 8 bytes no frame head
    fits: bytes whose every length word is negative."""
    if start < 8:
        return bytes(rng.randrange(0x80, 256) for _ in range(start))
    if start < 32:
        return (struct.pack(">ii", max(start + 3, 16), eu.NOTIFY_XID) + b"\xa5" * start)[:start]
    out = b""
    while start - len(out) >= 20 + 32:
        out += ru.ping()
    rest = start - len(out)
    ln = rest + 7 - 4
    head = struct.pack(">iiqiiii", ln, eu.NOTIFY_XID, -1, 0, eu.DATA_CHANGED, eu.SYNC_CONNECTED, ln - 28)
    return out + (head + b"\xa5" * rest)[:rest]
