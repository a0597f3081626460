"""An independent restatement of regk_dns_answer with REGK_DNS_PTR, on top of dns_util: the reverse map is taken from
the HOST_A presentation lines of the resolve_util restatement (parsed back from text), a reverse name is recognised
with a regular expression, and PTR responses are built RR by RR and cut by trying each RR in turn.  Every other
message, and every message without the flag, is dns_util.answer's."""
import re
import struct

import dns_util as du
import resolve_util as rv

T_PTR = 12
_OCTET = re.compile(rb"0|[1-9][0-9]{0,2}")


def reverse_addr(labels):
    """the dotted-quad text a reverse name o4.o3.o2.o1.in-addr.arpa asks about, or None"""
    if len(labels) != 6 or labels[4].lower() != b"in-addr" or labels[5].lower() != b"arpa":
        return None
    if not all(_OCTET.fullmatch(x) and int(x) <= 255 for x in labels[:4]):
        return None
    return b".".join(reversed(labels[:4]))


def reverse_name(addr: bytes) -> bytes:
    return b".".join(reversed(addr.split(b"."))) + b".in-addr.arpa"


def reverse_map(zone: du.Zone):
    """address text -> [(node, ttl, name)] in node order, from the HOST_A lines"""
    out = {}
    res = zone.resolved
    for q, (kind, j) in enumerate(zip(res["q_kind"], res["q_node"])):
        if kind != rv.HOST_A:
            continue
        owner, ttl, _, _, addr = res["sections"][q][0].rstrip(b"\n").split(b"\t")
        out.setdefault(addr, []).append((j, int(ttl), owner[:-1]))
    return out


def ptr_rr(ttl, name):
    w = du.wire_name(name)
    return struct.pack(">HHHIH", 0xC00C, T_PTR, 1, ttl, len(w)) + w


def answer(zone, msg, udp_payload=1232, tcp=False, ptr=True, rmap=None):
    """(status, tc, node, response bytes) for one message"""
    r = du.parse(msg)
    addr = reverse_addr(r["labels"]) if ptr and r["status"] == du.ANSWER else None
    if addr is None:
        return du.answer(zone, msg, udp_payload, tcp)
    targets = (reverse_map(zone) if rmap is None else rmap).get(addr, [])
    own_a, own_s = zone.owners(r["labels"])
    qtype = r["qtype"]
    if (qtype == du.T_A and own_a is not None) or (qtype == du.T_SRV and own_s is not None) or not targets:
        return du.answer(zone, msg, udp_payload, tcp)
    ident, flags = struct.unpack(">HH", msg[:4])
    opcode, rd = (flags >> 11) & 0xF, (flags >> 8) & 1
    qend = r["qend"]
    st, node, answers = du.NODATA, du.NONE, []
    if qtype == T_PTR:
        st, node = du.ANSWER, targets[0][0]
        answers = [ptr_rr(t, name) for _, t, name in targets]
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
    hdr = struct.pack(">HHHHHH", ident, 0x8000 | opcode << 11 | 1 << 10 | tc << 9 | rd << 8, 1, n_ans, 0,
                      1 if r["opt"] else 0)
    opt = b"\0" + struct.pack(">HHIH", du.T_OPT, udp_payload, r["do"] << 15, 0) if r["opt"] else b""
    return st, tc, node, hdr + msg[12:qend] + ans + opt


def answer_all(zone, msgs, udp_payload=1232, tcp=False, ptr=True):
    """dict of the arrays regk_dns_answer returns"""
    rmap = reverse_map(zone)
    out = [answer(zone, m, udp_payload, tcp, ptr, rmap) for m in msgs]
    resp_off = [0]
    for o in out:
        resp_off.append(resp_off[-1] + len(o[3]))
    n_status = [0] * 8
    for o in out:
        n_status[o[0]] += 1
    return dict(status=[o[0] for o in out], tc=[o[1] for o in out], node=[o[2] for o in out], resp_off=resp_off,
                resp=b"".join(o[3] for o in out), n_status=n_status, n_truncated=sum(o[1] for o in out))
