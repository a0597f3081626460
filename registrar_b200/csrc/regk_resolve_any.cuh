/*
 * regk_resolve_any.cuh — REGK_RESOLVE_ANY_FORM (include/regk.h): host and service records in any JSON form Binder
 * reads, for the nodes the canonical recogniser (regk_decode_core.cuh decode_payload) refuses.  Reference: README.md
 * :441-755 (records, "About TTLs" :670-755).
 *
 * The reader is host + device code (tests/emul/resolve_any_emul.cpp runs it under AddressSanitizer with every payload
 * flush against the end of its buffer).  It is a single-exit loop over the payload's tokens, in the style of
 * decode_payload: whitespace and string bodies are scanned in 4-byte windows (quote, backslash and control bytes; JSON
 * whitespace), a failed requirement latches the cursor's error and the loop runs to its common end.  Containers are
 * tracked by a 64-bit stack of kinds (object / array), so the 64-level limit costs one register; the role of each of the
 * first three levels (which inspected object it is) sits in 4 bits of another.  Every member of the four inspected
 * objects - the top object, top.service, top.service.service and the host's inner object top.<type> - has a slot:
 * 4 bits of kind in one 64-bit word, last wins, and a member that starts an inspected object clears the slots of the
 * object it replaces.
 * The member that names a host's inner object may come before "type": the reader makes a SECOND PASS over the payload
 * when the first one found a host record's type (payloads are a few hundred bytes, already in L1 from the first pass;
 * remembering every object-valued top-level member instead would cost a register set per candidate).  The first pass
 * fills the top, service and ttl slots; the second only the inner object's and its ports.
 *
 * The passes (regk_api.cu resolve_meta, between regk_decode_kernel and classify, with the flag only):
 *   any_count / any_compact  the candidates (non-empty data, DEC_PATH_OK, refused by decode_payload) in node order,
 *                            over the project's two-level totals; the host reads the count once
 *   any_read                 one thread per candidate: the reader, word loads, GUARD for a payload that ends within 16
 *                            bytes of json_limit (a device snapshot can end exactly at the caller's allocation)
 *   classify_any             classify, reading the reader's TTL presence bit (RV_DEC_TTL_IN) for the nodes it read
 */
#ifndef REGK_RESOLVE_ANY_CUH
#define REGK_RESOLVE_ANY_CUH

#include "regk_resolve.cuh"

namespace regk {

/* slots, 4 bits of kind each in AnyRec::st: the inspected members, the top object itself and a ports element */
enum : uint32_t { AS_TYPE, AS_TTL_TOP, AS_MID, AS_TTL_MID, AS_SIN, AS_SRVCE, AS_PROTO, AS_PORT, AS_TTL_SIN, AS_INNER, AS_ADDR,
                  AS_PORTS, AS_TTL_INNER, AS_TOP, AS_ELEM, AS_NONE };
enum : uint32_t { AK_ABSENT = 0, AK_OBJ = 1, AK_ARR = 2, AK_STR = 3, AK_INT = 4, AK_OTHER = 5 };
/* the inspected containers: top, top.service, top.service.service, top.<type>, top.<type>.ports */
enum : uint32_t { AR_NONE = 0, AR_TOP = 1, AR_MID = 2, AR_SIN = 3, AR_INNER = 4, AR_PORTS = 5 };
enum : uint32_t { AM_VALUE, AM_FIRST_VALUE, AM_NAME, AM_FIRST_NAME, AM_AFTER };
constexpr uint32_t ANY_MAX_DEPTH = 64;

struct AnyRec {
    uint64_t st;                                /* AK_* per slot */
    uint32_t tp, tl, sp, sl, pp, pl, ap, al;    /* type, srvce, proto and the inner address: position, length */
    int32_t t_top, t_mid, t_sin, t_inner;       /* the ttl members (meaningful when their slot is AK_INT) */
    uint32_t port, np;                          /* the service's port; elements of the last ports array */
    bool pbad;                                  /* the last ports array holds something other than a port */
};

RG_HD uint32_t any_kind(const AnyRec &r, uint32_t slot)
{
    return (uint32_t)(r.st >> (4u * slot)) & 15u;
}

/* a member of an inspected object starts: its kind, and the slots of the object it replaces are cleared */
RG_HD void any_put(AnyRec &r, uint32_t slot, uint32_t kind)
{
    const uint64_t kids = slot == AS_MID ? 0x0000000FFFFFF000ull : slot == AS_SIN ? 0x0000000FFFF00000ull :
                          slot == AS_INNER ? 0x000FFF0000000000ull : 0ull;
    r.st = (r.st & ~kids & ~(15ull << (4u * slot))) | ((uint64_t)kind << (4u * slot));
}

/* bit 7 of every byte of v that is zero, exactly */
RG_HD uint32_t zero_bytes_exact(uint32_t v)
{
    return ~(((v & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | v | 0x7F7F7F7Fu);
}

/* bytes [pos, pos + len) of the payload spell s */
template <bool GUARD, size_t N>
RG_HD bool any_name_is(const Cur<GUARD> &c, uint32_t pos, uint32_t len, const char (&s)[N])
{
    constexpr uint32_t L = (uint32_t)(N - 1);
    uint32_t diff = len != L ? 1u : 0u;
    #pragma unroll
    for (uint32_t k = 0; k + 4u <= L; k += 4u)
        diff |= c.peek(pos + k) ^ lit_word(s, k);
    if (L & 3u)
        diff |= (c.peek(pos + (L & ~3u)) ^ lit_word(s, L & ~3u)) & low_bytes(L & 3u);
    return diff == 0;
}

/* JSON whitespace (space, TAB, LF, CR), four bytes at a time */
template <bool GUARD>
RG_HD void any_ws(Cur<GUARD> &c)
{
    bool go = c.i < c.n;
    while (go) {
        const uint32_t w = c.peek(c.i);
        const uint32_t ws = zero_bytes_exact(w ^ 0x20202020u) | zero_bytes_exact(w ^ 0x09090909u) | zero_bytes_exact(w ^ 0x0A0A0A0Au) |
                            zero_bytes_exact(w ^ 0x0D0D0D0Du);
        const uint32_t other = ~ws & 0x80808080u;
        const uint32_t k = other ? ctz32(other) >> 3 : 4u;
        c.i += k;
        go = k == 4u && c.i < c.n;
    }
    c.i = c.i < c.n ? c.i : c.n;
}

RG_HD bool any_hex(uint32_t b)
{
    return (b >= '0' && b <= '9') || ((b | 0x20u) >= 'a' && (b | 0x20u) <= 'f');
}

/* a string body after its opening quote, RFC 8259: no control bytes, escapes \" \\ \/ \b \f \n \r \t \uXXXX (kept as they
   are).  [pos, pos + len) is the body; *esc: it holds an escape.  false: not a string */
template <bool GUARD>
RG_HD bool any_str(Cur<GUARD> &c, uint32_t *pos, uint32_t *len, bool *esc)
{
    *pos = c.i;
    *esc = false;
    uint32_t state = 0;                                         /* 0 scanning, 1 closing quote found, 2 not a string */
    while (state == 0) {
        if (c.i >= c.n) {
            state = 2;
        } else {
            const uint32_t w = c.peek(c.i);
            const uint32_t quote = zero_bytes_exact(w ^ 0x22222222u), back = zero_bytes_exact(w ^ 0x5C5C5C5Cu);
            const uint32_t ctl = ~(((w & 0x7F7F7F7Fu) + 0x60606060u) | w) & 0x80808080u;      /* bytes below 0x20 */
            const uint32_t m = quote | back | ctl;
            if (m == 0) {
                c.i += 4;
            } else {
                const uint32_t bit = ctz32(m);
                c.i += bit >> 3;
                if (c.i >= c.n || ((ctl >> bit) & 1u)) {
                    state = 2;
                } else if ((quote >> bit) & 1u) {
                    state = 1;
                } else {
                    *esc = true;
                    const uint32_t e = c.i + 1u < c.n ? c.byte_at(c.i + 1u) : 0u;
                    if (e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't') {
                        c.i += 2;
                    } else if (e == 'u' && c.i + 6u <= c.n) {
                        const uint32_t h = c.peek(c.i + 2u);
                        const bool ok = any_hex(h & 0xFFu) && any_hex((h >> 8) & 0xFFu) && any_hex((h >> 16) & 0xFFu) && any_hex(h >> 24);
                        c.i += ok ? 6u : 0u;
                        state = ok ? 0u : 2u;
                    } else {
                        state = 2;
                    }
                }
            }
        }
    }
    c.i = c.i < c.n ? c.i : c.n;
    *len = c.i - *pos;
    c.i += state == 1 ? 1u : 0u;
    return state == 1;
}

/* a run of decimal digits: their count; the value of the first 12 accumulates into *a */
template <bool GUARD>
RG_HD uint32_t any_digits(Cur<GUARD> &c, unsigned long long *a)
{
    uint32_t k = 0;
    bool go = true;
    while (go) {
        const uint32_t d = c.i < c.n ? c.byte_at(c.i) - (uint32_t)'0' : 10u;
        go = d <= 9u;
        if (go) {
            *a = k < 12u ? *a * 10u + d : *a;
            k++;
            c.i++;
        }
    }
    return k;
}

/* a JSON number; *kind = AK_INT when it is -?(0|[1-9][0-9]*), not -0, below 10^12 in magnitude (value in *v),
   AK_OTHER for every other number.  false: not a number */
template <bool GUARD>
RG_HD bool any_num(Cur<GUARD> &c, uint32_t *kind, long long *v)
{
    const bool neg = c.eat('-');
    const uint32_t d0 = c.i;
    unsigned long long a = 0, x = 0;
    const uint32_t k = any_digits(c, &a);
    bool ok = k != 0 && !(k > 1u && c.byte_at(d0) == '0');
    bool integral = true;
    if (c.eat('.')) {
        integral = false;
        ok = ok && any_digits(c, &x) != 0;
    }
    if (c.i < c.n && (c.byte_at(c.i) | 0x20u) == 'e') {
        integral = false;
        c.i++;
        if (!c.eat('+'))
            c.eat('-');
        ok = ok && any_digits(c, &x) != 0;
    }
    *kind = integral && k < 12u && !(neg && a == 0) ? AK_INT : AK_OTHER;
    *v = neg ? -(long long)a : (long long)a;
    return ok;
}

/* the slot of member [pos, pos + len) of a container of role `role`; pass 2 looks for the inner object only */
template <bool GUARD>
RG_HD uint32_t any_slot(const Cur<GUARD> &c, const AnyRec &r, uint32_t role, uint32_t pos, uint32_t len, bool pass2)
{
    uint32_t s = AS_NONE;
    if (role == AR_TOP && pass2)
        s = len == r.tl && same_bytes(c, pos, r.tp, len) ? AS_INNER : AS_NONE;
    else if (role == AR_TOP)
        s = any_name_is(c, pos, len, "type") ? AS_TYPE : any_name_is(c, pos, len, "ttl") ? AS_TTL_TOP :
            any_name_is(c, pos, len, "service") ? AS_MID : AS_NONE;
    else if (role == AR_MID)
        s = any_name_is(c, pos, len, "service") ? AS_SIN : any_name_is(c, pos, len, "ttl") ? AS_TTL_MID : AS_NONE;
    else if (role == AR_SIN)
        s = any_name_is(c, pos, len, "srvce") ? AS_SRVCE : any_name_is(c, pos, len, "proto") ? AS_PROTO :
            any_name_is(c, pos, len, "port") ? AS_PORT : any_name_is(c, pos, len, "ttl") ? AS_TTL_SIN : AS_NONE;
    else if (role == AR_INNER)
        s = any_name_is(c, pos, len, "address") ? AS_ADDR : any_name_is(c, pos, len, "ports") ? AS_PORTS :
            any_name_is(c, pos, len, "ttl") ? AS_TTL_INNER : AS_NONE;
    return s;
}

/* one pass over the whole payload: grammar, depth, raw member names; the slots of the inspected objects.  Ports of the
   inner object go to ports[] as they are read (an element costs >= 2 payload bytes, so n / 2 slots bound them). */
template <bool GUARD>
RG_HD void any_pass(Cur<GUARD> &c, AnyRec &r, uint32_t *ports, bool pass2)
{
    uint64_t arr = 0;                                           /* bit d - 1: the container at depth d is an array */
    uint32_t depth = 0, roles = 0;                              /* roles: AR_* of depths 1..3, 4 bits each */
    uint32_t mode = AM_VALUE, slot = AS_TOP;
    c.i = 0;
    any_ws(c);
    c.need(c.i < c.n && c.byte_at(c.i) == '{');                 /* the payload is one object */
    bool done = false;
    while (!done && !c.err) {
        any_ws(c);
        const uint32_t b = c.i < c.n ? c.byte_at(c.i) : 0x100u;
        const uint32_t role = depth - 1u < 3u ? (roles >> (4u * (depth - 1u))) & 15u : (uint32_t)AR_NONE;
        const bool in_arr = depth && ((arr >> ((depth - 1u) & 63u)) & 1u);
        if (mode == AM_AFTER) {
            if (depth == 0) {
                done = true;
            } else if (b == ',') {
                c.i++;
                mode = in_arr ? AM_VALUE : AM_NAME;
                slot = role == AR_PORTS ? AS_ELEM : AS_NONE;
            } else {
                c.need(b == (in_arr ? ']' : '}'));
                c.i++;
                depth--;
            }
        } else if ((mode == AM_FIRST_NAME && b == '}') || (mode == AM_FIRST_VALUE && b == ']')) {
            c.i++;
            depth--;
            mode = AM_AFTER;
        } else if (mode == AM_NAME || mode == AM_FIRST_NAME) {
            uint32_t pos = 0, len = 0;
            bool esc = false;
            c.need(b == '"');
            c.i++;
            c.need(any_str(c, &pos, &len, &esc) && !esc);       /* an escaped name could decode to an inspected one */
            any_ws(c);
            c.need(c.eat(':'));
            slot = c.err ? (uint32_t)AS_NONE : any_slot(c, r, role, pos, len, pass2);
            mode = AM_VALUE;
        } else if (b == '{' || b == '[') {
            const bool obj = b == '{';
            depth++;
            c.need(depth <= ANY_MAX_DEPTH);
            c.i++;
            const uint64_t bit = 1ull << ((depth - 1u) & 63u);
            arr = obj ? arr & ~bit : arr | bit;
            const uint32_t cr = obj ? (slot == AS_TOP ? AR_TOP : slot == AS_MID ? AR_MID : slot == AS_SIN ? AR_SIN :
                                       slot == AS_INNER ? AR_INNER : AR_NONE) : (slot == AS_PORTS ? AR_PORTS : AR_NONE);
            if (depth <= 3u)
                roles = (roles & ~(15u << (4u * (depth - 1u)))) | (cr << (4u * (depth - 1u)));
            if (slot == AS_PORTS) {
                r.np = 0;
                r.pbad = false;
            }
            if (slot == AS_ELEM)
                r.pbad = true;
            else
                any_put(r, slot, obj ? AK_OBJ : AK_ARR);
            mode = obj ? AM_FIRST_NAME : AM_FIRST_VALUE;
            slot = cr == AR_PORTS ? AS_ELEM : AS_NONE;
        } else {
            uint32_t kind = AK_OTHER, pos = 0, len = 0;
            long long v = 0;
            bool esc = false;
            if (b == '"') {
                c.i++;
                c.need(any_str(c, &pos, &len, &esc));
                kind = AK_STR;
            } else if (b == '-' || (b >= '0' && b <= '9')) {
                c.need(any_num(c, &kind, &v));
            } else if (b == 't') {
                c.need(c.lit("true"));
            } else if (b == 'f') {
                c.need(c.lit("false"));
            } else {
                c.need(b == 'n' && c.lit("null"));
            }
            const bool ttl = slot == AS_TTL_TOP || slot == AS_TTL_MID || slot == AS_TTL_SIN || slot == AS_TTL_INNER;
            if (kind == AK_INT && !(ttl ? v >= -2147483648ll && v <= 2147483647ll : v >= 0 && v <= 4294967295ll))
                kind = AK_OTHER;
            if (slot == AS_ELEM) {
                if (kind == AK_INT && !r.pbad && !c.err)
                    ports[r.np++] = (uint32_t)v;
                r.pbad = r.pbad || kind != AK_INT;
            } else {
                any_put(r, slot, kind);
            }
            r.tp = slot == AS_TYPE ? pos : r.tp;
            r.tl = slot == AS_TYPE ? len : r.tl;
            r.sp = slot == AS_SRVCE ? pos : r.sp;
            r.sl = slot == AS_SRVCE ? len : r.sl;
            r.pp = slot == AS_PROTO ? pos : r.pp;
            r.pl = slot == AS_PROTO ? len : r.pl;
            r.ap = slot == AS_ADDR ? pos : r.ap;
            r.al = slot == AS_ADDR ? len : r.al;
            r.t_top = slot == AS_TTL_TOP ? (int32_t)v : r.t_top;
            r.t_mid = slot == AS_TTL_MID ? (int32_t)v : r.t_mid;
            r.t_sin = slot == AS_TTL_SIN ? (int32_t)v : r.t_sin;
            r.t_inner = slot == AS_TTL_INNER ? (int32_t)v : r.t_inner;
            r.port = slot == AS_PORT ? (uint32_t)v : r.port;
            mode = AM_AFTER;
        }
    }
    any_ws(c);
    c.need(c.i == c.n);                                         /* nothing but whitespace behind the object */
}

/* RV_DEC_ANY_READ / RV_DEC_TTL_IN: internal bits of Decoded.flags above the public REGK_DEC_* (never returned by
   regk_decode); regk_resolve.cuh rv_classify<true> reads them */

/* The general reader on payload [p, p + n) of a candidate node (d: its regk_decode record).  On success d becomes the
   record in the layout classify reads - service: type = srvce, addr = proto, ports[0] = port, nports = 1; host: type,
   addr = the inner address, its ports (nports ~0 without a ports member) - with d.ttl the TTL the README's precedence
   picks and RV_DEC_TTL_IN when there is one.  On failure d is left as it is (the node stays REGK_RSV_NOT_RECORD). */
template <bool GUARD>
RG_HD bool read_any(const uint8_t *p, uint32_t n, Decoded &d, uint32_t *ports)
{
    Cur<GUARD> c;
    c.init(p, n);
    AnyRec r;
    r.st = 0;
    r.tp = r.tl = r.sp = r.sl = r.pp = r.pl = r.ap = r.al = 0;
    r.t_top = r.t_mid = r.t_sin = r.t_inner = 0;
    r.port = r.np = 0;
    r.pbad = false;
    bool typed = false, svc = false;
    uint32_t pass = 0;
    bool again = true;
    while (again) {                                             /* one copy of the pass in the code, run once or twice */
        any_pass(c, r, ports, pass != 0);
        if (pass == 0) {
            typed = !c.err && any_kind(r, AS_TYPE) == AK_STR;
            svc = typed && any_name_is(c, r.tp, r.tl, "service");
        }
        again = pass == 0 && typed && !svc;
        pass++;
    }
    const uint32_t k_top = any_kind(r, AS_TTL_TOP), k_mid = any_kind(r, AS_TTL_MID), k_sin = any_kind(r, AS_TTL_SIN),
                   k_inner = any_kind(r, AS_TTL_INNER);
    bool ok = typed && !c.err && (k_top == AK_ABSENT || k_top == AK_INT);
    int32_t ttl = INT32_MIN;
    bool ttl_in = false;
    if (svc) {
        ok = ok && any_kind(r, AS_MID) == AK_OBJ && any_kind(r, AS_SIN) == AK_OBJ && any_kind(r, AS_SRVCE) == AK_STR &&
             any_kind(r, AS_PROTO) == AK_STR && any_kind(r, AS_PORT) == AK_INT && (k_mid == AK_ABSENT || k_mid == AK_INT) &&
             (k_sin == AK_ABSENT || k_sin == AK_INT);
        ttl_in = k_sin == AK_INT || k_mid == AK_INT || k_top == AK_INT;
        ttl = k_sin == AK_INT ? r.t_sin : k_mid == AK_INT ? r.t_mid : k_top == AK_INT ? r.t_top : INT32_MIN;
    } else {
        const uint32_t kp = any_kind(r, AS_PORTS);
        ok = ok && any_kind(r, AS_INNER) == AK_OBJ && any_kind(r, AS_ADDR) == AK_STR && (kp == AK_ABSENT || (kp == AK_ARR && !r.pbad)) &&
             (k_inner == AK_ABSENT || k_inner == AK_INT);
        ttl_in = k_inner == AK_INT || k_top == AK_INT;
        ttl = k_inner == AK_INT ? r.t_inner : k_top == AK_INT ? r.t_top : INT32_MIN;
    }
    if (ok) {
        d.flags = (d.flags & DEC_PATH_OK) | (svc ? DEC_SERVICE_RECORD : DEC_HOST_RECORD) | RV_DEC_ANY_READ | (ttl_in ? RV_DEC_TTL_IN : 0u);
        d.type_pos = svc ? r.sp : r.tp;
        d.type_len = svc ? r.sl : r.tl;
        d.addr_pos = svc ? r.pp : r.ap;
        d.addr_len = svc ? r.pl : r.al;
        d.ttl = ttl;
        d.nports = svc ? 1u : any_kind(r, AS_PORTS) == AK_ARR ? r.np : 0xFFFFFFFFu;
        if (svc)
            ports[0] = r.port;
    }
    return ok;
}

/* a node the general reader decides: non-empty data, a path, and a class of REGK_RSV_NOT_RECORD from regk_decode's record */
RG_HD bool any_candidate(const Decoded &d, uint64_t jn)
{
    const uint32_t bad = DEC_NOT_CANONICAL | DEC_KEY_MISMATCH | DEC_ADDR_MISMATCH | DEC_BAD_NUMBER | DEC_BAD_PATH;
    return jn != 0 && (d.flags & DEC_PATH_OK) && ((d.flags & bad) || !(d.flags & (DEC_HOST_RECORD | DEC_SERVICE_RECORD)));
}

}  /* namespace regk */

#if defined(__CUDACC__)
namespace regk {

struct AnyParams {
    uint64_t m;
    const uint8_t *json;
    const unsigned long long *json_off;
    uint64_t json_limit;                        /* bytes readable behind the data stream */
    Decoded *dec;
    uint32_t *ports;
    uint32_t *list;                             /* [m] the candidates, ascending */
    unsigned long long *tile_total[3], *super_total[3];   /* [0]: the candidates per tile (the others unused) */
    unsigned long long *count;                  /* the number of candidates */
};

/* ---- any_count: candidates per tile ---- */
__global__ void __launch_bounds__(RV_TILE) regk_resolve_any_count_kernel(const AnyParams p)
{
    const uint64_t j = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long v[1] = {0ull}, tot[1];
    if (j < p.m)
        v[0] = any_candidate(p.dec[j], p.json_off[j + 1] - p.json_off[j]) ? 1ull : 0ull;
    rv_block_scan<1>(v, tot);
    if (threadIdx.x == 0)
        rv_add_total(p.tile_total[0], p.super_total[0], blockIdx.x, tot[0]);
}

/* ---- any_compact: the candidates in node order, and their count ---- */
__global__ void __launch_bounds__(RV_TILE) regk_resolve_any_compact_kernel(const AnyParams p)
{
    const uint64_t j = (uint64_t)blockIdx.x * RV_TILE + threadIdx.x;
    unsigned long long base[1], v[1] = {0ull}, tot[1];
    rv_tile_bases<1>(p.tile_total, p.super_total, blockIdx.x, base);
    const bool cand = j < p.m && any_candidate(p.dec[j], p.json_off[j + 1] - p.json_off[j]);
    v[0] = cand ? 1ull : 0ull;
    rv_block_scan<1>(v, tot);
    if (cand)
        p.list[base[0] + v[0]] = (uint32_t)j;
    if (j + 1 == p.m)
        *p.count = base[0] + v[0] + (cand ? 1ull : 0ull);
}

/* ---- any_read: one thread per candidate (a minimum of one CTA per SM: ptxas' own occupancy target capped the kernel
   at 64 registers and spilled; it takes 80 without the cap) ---- */
__global__ void __launch_bounds__(256, 1) regk_resolve_any_read_kernel(const AnyParams p, uint32_t n_cand)
{
    const uint32_t t = blockIdx.x * 256u + threadIdx.x;
    if (t >= n_cand)
        return;
    const uint32_t j = p.list[t];
    const unsigned long long q0 = p.json_off[j], q1 = p.json_off[j + 1];
    Decoded d = p.dec[j];
    uint32_t *ports = p.ports + (q0 >> 1);
    /* word loads read up to 11 bytes behind a payload's end: bounded byte loads near the end of the stream */
    const bool ok = q1 + 16u <= p.json_limit ? read_any<false>(p.json + q0, (uint32_t)(q1 - q0), d, ports)
                                             : read_any<true>(p.json + q0, (uint32_t)(q1 - q0), d, ports);
    if (ok)
        p.dec[j] = d;
}

/* ---- classify with REGK_RESOLVE_ANY_FORM: the TTL presence of a node the general reader read is its bit ---- */
__global__ void __launch_bounds__(256) regk_resolve_classify_any_kernel(const ResolveParams p)
{
    rv_classify_node<true>(p);
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_RESOLVE_ANY_CUH */
