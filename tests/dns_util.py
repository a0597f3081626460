"""An independent restatement of regk_dns_answer, written from RFC 1035 / 2782 / 6891 and the rules in include/regk.h:
byte-by-byte parsing with struct, a dict of snapshot paths for the lookup, and the answer sets taken from the
presentation lines of the resolve_util restatement (parsed back from text).  Responses are built RR by RR and cut by
trying each RR in turn."""
import socket
import struct

import resolve_util as rv

ANSWER, NODATA, NXDOMAIN, FORMERR, NOTIMP, REFUSED, BADVERS, DROPPED = range(8)
PLAIN = set(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_-")
T_A, T_SRV, T_AAAA, T_OPT, T_ANY = 1, 33, 28, 41, 255
NONE = 2 ** 64 - 1


def parse(msg: bytes):
    """rules 1-8: dict(status, labels, qend, qtype, qclass, opt, do, req); status ANSWER means "look it up" """
    r = dict(status=FORMERR, labels=[], qend=0, qtype=0, qclass=0, opt=False, do=0, req=0)
    if len(msg) < 12 or msg[2] & 0x80:
        r["status"] = DROPPED
        return r
    if (msg[2] >> 3) & 0xF:
        r["status"] = NOTIMP
        return r
    _, _, qd, an, ns, ar = struct.unpack(">HHHHHH", msg[:12])
    if qd != 1 or an or ns or ar > 1:
        return r
    pos, labels = 12, []
    while True:
        if pos >= len(msg):
            return r
        n = msg[pos]
        if n & 0xC0:
            return r
        pos += 1
        if n == 0:
            break
        if pos + n > len(msg):
            return r
        labels.append(msg[pos:pos + n])
        pos += n
    if pos - 12 > 255 or pos + 4 > len(msg):
        return r
    r["labels"] = labels
    r["qtype"], r["qclass"] = struct.unpack(">HH", msg[pos:pos + 4])
    pos += 4
    r["qend"] = pos
    version = 0
    if ar:
        if pos + 11 > len(msg) or msg[pos] != 0:
            return r
        typ, cls, ttl, rdlen = struct.unpack(">HHIH", msg[pos + 1:pos + 11])
        if typ != T_OPT:
            return r
        pos += 11 + rdlen
        if pos > len(msg):
            return r
        r.update(opt=True, req=cls, do=(ttl >> 15) & 1)
        version = (ttl >> 16) & 0xFF
    if pos != len(msg):
        return r
    r["status"] = BADVERS if version else REFUSED if r["qclass"] != 1 else ANSWER
    return r


def _lines(text: bytes):
    return [ln.split(b"\t") for ln in text.splitlines()]


class Zone:
    """What a snapshot answers, from rv.resolve: per node its A answers, per service node its SRV answers and
    additionals, and srvce / proto"""

    def __init__(self, nodes, dh=30, ds=60):
        res = rv.resolve(nodes, dh, ds)
        self.index = {p: j for j, (p, _) in enumerate(nodes)}
        self.a, self.srv, self.rec = {}, {}, {}
        for q, (kind, j) in enumerate(zip(res["q_kind"], res["q_node"])):
            ans, add = res["sections"][q]
            if kind == rv.SERVICE_SRV:
                srv = [(int(t), int(rd.split(b" ")[2]), rd.split(b" ")[3][:-1]) for _, t, _, _, rd in _lines(ans)]
                extra = [(o[:-1], int(t), a) for o, t, _, _, a in _lines(add)]
                self.srv[j] = (srv, extra)
                self.rec[j] = rv.classify(*nodes[j])[1]
            else:
                self.a[j] = (kind, [(int(t), a) for _, t, _, _, a in _lines(ans)])
        self.resolved = res

    def node(self, labels):
        if not labels or any(c not in PLAIN for lab in labels for c in lab):
            return None
        return self.index.get(b"/" + b"/".join(lab.lower() for lab in reversed(labels)))

    def owners(self, labels):
        """(node owning A or None, service node owning SRV or None)"""
        j = self.node(labels)
        own_a = j if j in self.a else None
        own_s = None
        if len(labels) >= 3:
            s = self.node(labels[2:])
            if s in self.srv:
                _, srvce, proto, _, _ = self.rec[s]
                if labels[0].lower() == srvce.lower() and labels[1].lower() == proto.lower():
                    own_s = s
        return own_a, own_s


def a_rr(owner_ptr, ttl, addr):
    return struct.pack(">HHHIH", 0xC000 | owner_ptr, T_A, 1, ttl, 4) + socket.inet_aton(addr.decode())


def wire_name(name: bytes):
    return b"".join(bytes([len(x)]) + x for x in name.split(b".")) + b"\0"


def srv_rr(ttl, port, target):
    rdata = struct.pack(">HHH", 0, 10, port) + wire_name(target)
    return struct.pack(">HHHIH", 0xC00C, T_SRV, 1, ttl, len(rdata)) + rdata


def answer(zone: Zone, msg: bytes, udp_payload=1232, tcp=False):
    """(status, tc, node, response bytes) for one message"""
    r = parse(msg)
    st = r["status"]
    if st == DROPPED:
        return st, 0, NONE, b""
    ident, flags = struct.unpack(">HH", msg[:4])
    opcode, rd = (flags >> 11) & 0xF, (flags >> 8) & 1
    if st in (FORMERR, NOTIMP):
        rcode = 1 if st == FORMERR else 4
        return st, 0, NONE, struct.pack(">HHHHHH", ident, 0x8000 | opcode << 11 | rd << 8 | rcode, 0, 0, 0, 0)
    node, answers, extra = NONE, [], []
    qend = r["qend"]
    if st == ANSWER:
        own_a, own_s = zone.owners(r["labels"])
        if r["qtype"] == T_A and own_a is not None:
            node = own_a
            answers = [a_rr(12, t, a) for t, a in zone.a[own_a][1]]
        elif r["qtype"] == T_SRV and own_s is not None:
            node = own_s
            srv, add = zone.srv[own_s]
            first, off = {}, qend
            for t, p, target in srv:
                first.setdefault(target, off)
                rr = srv_rr(t, p, target)
                answers.append(rr)
                off += len(rr)
            extra = [(first[o] + 18, a_rr(first[o] + 18 if first[o] + 18 < 0x4000 else 0, t, a)) for o, t, a in add]
        else:
            st = NODATA if (own_a is not None or own_s is not None) else NXDOMAIN
    limit = 65535 if tcp else (min(max(r["req"], 512), udp_payload) if r["opt"] else 512)
    size = qend + (11 if r["opt"] else 0)
    ans, n_ans = b"", 0
    for rr in answers:
        if size + len(rr) > limit:
            break
        ans += rr
        size += len(rr)
        n_ans += 1
    tc = int(n_ans < len(answers))
    add, n_add = b"", 0
    if not tc:
        for ptr, rr in extra:
            if ptr > 0x3FFF or size + len(rr) > limit:
                break
            add += rr
            size += len(rr)
            n_add += 1
    rcode = {NXDOMAIN: 3, REFUSED: 5}.get(st, 0)
    aa = 1 if st in (ANSWER, NODATA, NXDOMAIN) else 0
    hdr = struct.pack(">HHHHHH", ident, 0x8000 | opcode << 11 | aa << 10 | tc << 9 | rd << 8 | rcode, 1, n_ans, 0,
                      n_add + (1 if r["opt"] else 0))
    opt = b""
    if r["opt"]:
        opt = b"\0" + struct.pack(">HHIH", T_OPT, udp_payload, (1 << 24 if st == BADVERS else 0) | r["do"] << 15, 0)
    return st, tc, node, hdr + msg[12:qend] + ans + add + opt


def answer_all(zone, msgs, udp_payload=1232, tcp=False):
    """dict of the arrays regk_dns_answer returns"""
    out = [answer(zone, m, udp_payload, tcp) for m in msgs]
    resp_off = [0]
    for o in out:
        resp_off.append(resp_off[-1] + len(o[3]))
    n_status = [0] * 8
    for o in out:
        n_status[o[0]] += 1
    return dict(status=[o[0] for o in out], tc=[o[1] for o in out], node=[o[2] for o in out], resp_off=resp_off,
                resp=b"".join(o[3] for o in out), n_status=n_status, n_truncated=sum(o[1] for o in out))


def query(name: bytes, qtype=T_A, ident=0x1234, rd=1, opcode=0, qclass=1, opt=None, extra=b""):
    """a query message; opt = (udp size, version, do) adds an OPT record"""
    q = wire_name(name) if name else b"\0"
    ar = 1 if opt is not None else 0
    msg = struct.pack(">HHHHHH", ident, opcode << 11 | rd << 8, 1, 0, 0, ar) + q + struct.pack(">HH", qtype, qclass)
    if opt is not None:
        size, version, do = opt
        msg += b"\0" + struct.pack(">HHIH", T_OPT, size, version << 16 | do << 15, 0)
    return msg + extra


def pack(msgs):
    """(bytes as uint8 array, int64 offsets)"""
    import numpy as np
    off = np.zeros(len(msgs) + 1, np.int64)
    np.cumsum([len(m) for m in msgs], out=off[1:])
    return np.frombuffer(b"".join(msgs), np.uint8).copy(), off
