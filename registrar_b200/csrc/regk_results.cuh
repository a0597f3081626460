/*
 * regk_results.cuh — read ZooKeeper's replies to the write frames this library made (regk_jute_frames /
 * regk_jute_requests with create, delete or setData; regk_mkdirp_requests; regk_reconcile_requests; the stale deletes of
 * regk_children_requests) and say, per list entry, whether its write took effect.  The reference learns the outcome of
 * each write from its callback (lib/register.js:85-95 ignores NO_NODE on the unlink, zkplus' mkdirp ignores
 * NODE_EXISTS); a registrar that frames a whole fleet's writes reads the whole reply stream at once instead.
 *
 * PARITY UNPINNED: the layouts below are restated from zookeeper.jute (ReplyHeader, CreateResponse, SetDataResponse,
 * Stat, MultiHeader, ErrorResponse) and from the server's multi handling (FinalRequestProcessor, DataTree), and tested
 * against an independent restatement, not against a server.  Big endian throughout.
 *   frame        int len | ReplyHeader{int xid; long zxid; int err} | body            (20 bytes before the body)
 *   create       err == 0: CreateResponse{int P | P path bytes}, len == 20 + P; the path is the framed one, byte for byte
 *   delete       len == 16
 *   setData      err == 0: Stat (68 bytes), len == 84; Stat.version at +32, Stat.dataLength (== the framed data's length)
 *                at +52
 *   error        err != 0: len == 16, no body (a multi with err != 0 fails every operation of its frame with err)
 *   multi        err == 0: MultiResponse = per operation MultiHeader{int type; bool done = 0; int err} + result, then
 *                MultiHeader{-1, 1, -1}.  Applied: typed results (type = the framed op, err 0): create 4 + P bytes, delete
 *                none, setData a Stat.  Rolled back: only ErrorResults, MultiHeader{-1, 0, e} + ErrorResponse{int e}, 13
 *                bytes each; the operations before the failing one carry 0, the failing one its code, those after it -2
 *                (RUNTIMEINCONSISTENCY).
 * A frame of m operations over the entries [a, b) therefore has exactly two success lengths, closed form in the framed
 * path lengths (sum P = path_off[b] - path_off[a]):
 *   applied      25 + 13m + sum P (create), 25 + 9m (delete), 25 + 77m (setData), 25 + 22e + sum P (replace, e entries)
 *   rolled back  25 + 13m
 * The length decides the outcome; where both are equal (a replace whose paths average 4 bytes) the first MultiHeader's
 * type does.  Each entry's result then sits at a closed-form position: frame + 20 + i x (13 | 9 | 77 | 22) + the framed
 * path bytes of the entries before it (applied), frame + 20 + 13 x its operation index (rolled back).  Only the frames
 * are a chain; entries need none.
 *
 * results_head() is the plausibility test of one position, results_check() the frame check of reply k, results_entry()
 * the check and outcome of one entry; all three are host + device code (the CPU tests run them).
 *
 * The passes:
 *   frames   cand (results_head() at every position at or after start: an in-range xid fixes frame k and with it the
 *            two or three lengths its reply can have), then regk_replies.cuh's compact, succ, jump and mark kernels and
 *            its chain count; the chain kernel here checks reply k < frames against xid_base + k and records its
 *            position and err.
 *   entries  one thread per entry of the frames before the first frame fault: results_entry() at its closed-form
 *            position; err, class, version and subject per entry, per-CTA counts of FAILED and ABORTED entries into
 *            two-level totals.
 *   lists    the FAILED and ABORTED entries compacted, ascending.
 */
#ifndef REGK_RESULTS_CUH
#define REGK_RESULTS_CUH

#include "regk_replies.cuh"

namespace regk {

/* results_head / results_check / results_entry results */
enum : uint32_t {
    RS_OK = 0,
    RS_TRUNC,           /* the stream ends inside the frame (or before its length word) */
    RS_BAD_LEN,         /* len < 16: no room for a ReplyHeader */
    RS_NEG_XID,         /* a negative xid other than -1 / -2 */
    RS_XID_RANGE,       /* an xid outside [xid_base, xid_base + frames) */
    RS_ERR_BODY,        /* err != 0 and a body */
    RS_SUCC_LEN,        /* err == 0 and a length that fits neither outcome of the frame */
    RS_ORDER,           /* an xid in range but not xid_base + k */
    RS_OP_TYPE,         /* a MultiHeader that is not {framed op, 0, 0} of an applied multi or {-1, 0, e} of a rolled-back one */
    RS_PATH_ECHO,       /* a CreateResponse path that differs from the framed path */
    RS_STAT_LEN,        /* a setData Stat.dataLength that differs from the framed data's length */
    RS_ERR_RESULT,      /* an ErrorResult whose ErrorResponse differs from its header's err */
    RS_ERR_SEQ,         /* ErrorResults that are not 0 .. 0, the failing code, -2 .. -2 */
    RS_CLOSE,           /* a multi's closing MultiHeader{-1, true, -1} is missing */
    RS_NO_FAILURE,      /* a rolled-back multi whose ErrorResults are all 0 */
};

/* cls[] (include/regk.h REGK_RES_DONE / _FAILED / _ABORTED) */
enum : uint8_t { RS_DONE = 0, RS_FAILED = 1, RS_ABORTED = 2 };

constexpr uint32_t RS_REPLACE = 256u;           /* ResFraming::op of a replace framing (REGK_ZK_REPLACE) */

/* What one write framing framed: frame k holds entries [k g, min((k + 1) g, entries)); entry e's path is
   path_bytes[path_off[e], path_off[e + 1]) and, for setData, its data is data_off[e + 1] - data_off[e] bytes. */
struct ResFraming {
    int32_t xid_base;
    uint32_t op;                                /* 1 create, 2 delete, 5 setData, RS_REPLACE */
    uint32_t group;                             /* entries per frame, >= 1 */
    uint32_t multi;                             /* frames are multi transactions */
    uint64_t frames, entries;
    const uint8_t *path_bytes;
    const unsigned long long *path_off;         /* [entries + 1] */
    const unsigned long long *data_off;         /* [entries + 1] for setData, else unused */
};

struct ResHead {
    uint32_t kind;      /* RK_* */
    int32_t len, xid, err;
};

RG_HD uint32_t rs_ops(const ResFraming &f)
{
    return f.op == RS_REPLACE ? 2u : 1u;
}

/* the bytes one entry's typed results take in an applied multi, not counting its path */
RG_HD uint32_t rs_fixed(const ResFraming &f)
{
    return f.op == 1u ? 13u : f.op == 2u ? 9u : f.op == 5u ? 77u : 22u;
}

/* the length word of frame k's reply when its writes took effect (*ok) or were rolled back (*bad; multi only) */
RG_HD void rs_lens(const ResFraming &f, uint64_t k, int64_t *ok, int64_t *bad)
{
    const uint64_t a = k * f.group, b = a + f.group < f.entries ? a + f.group : f.entries;
    const int64_t P = (int64_t)(f.path_off[b] - f.path_off[a]);
    if (!f.multi) {
        *ok = f.op == 1u ? 20 + P : f.op == 2u ? 16 : 84;
        *bad = -1;
        return;
    }
    const int64_t m = (int64_t)(b - a);
    *ok = 25 + (int64_t)rs_fixed(f) * m + (f.op == 1u || f.op == RS_REPLACE ? P : 0);
    *bad = 25 + 13 * m * (int64_t)rs_ops(f);
}

/* Plausibility of a frame starting at b, with `avail` stream bytes from b on (reads at most 20 of them, never past
   avail): the frame fits, its xid is -1, -2 or one of the framed requests', an error has len 16 and a success one of
   the lengths its frame's reply can have. */
RG_HD uint32_t results_head(const uint8_t *b, uint64_t avail, const ResFraming &f, ResHead *h)
{
    h->kind = RK_REPLY;
    h->len = h->xid = h->err = 0;
    if (avail < 4)
        return RS_TRUNC;
    const int32_t L = (int32_t)be32_at(b);
    h->len = L;
    if (L < 16)
        return RS_BAD_LEN;
    if ((uint64_t)L + 4u > avail)
        return RS_TRUNC;
    const int32_t xid = (int32_t)be32_at(b + 4), err = (int32_t)be32_at(b + 16);
    h->xid = xid;
    h->err = err;
    if (xid == -1 || xid == -2) {
        h->kind = xid == -1 ? RK_NOTIFY : RK_PING;
        return RS_OK;
    }
    const uint64_t k = (uint32_t)xid - (uint32_t)f.xid_base;
    if (k >= f.frames)
        return xid < 0 ? RS_NEG_XID : RS_XID_RANGE;
    if (err != 0)
        return L == 16 ? RS_OK : RS_ERR_BODY;
    int64_t ok, bad;
    rs_lens(f, k, &ok, &bad);
    return L == ok || L == bad ? RS_OK : RS_SUCC_LEN;
}

/* results_head(), then the xid against xid_base + k.  Notifications and pings pass with their kind set. */
RG_HD uint32_t results_check(const uint8_t *b, uint64_t avail, const ResFraming &f, uint64_t k, ResHead *h)
{
    const uint32_t c = results_head(b, avail, f, h);
    if (c != RS_OK || h->kind != RK_REPLY)
        return c;
    if ((uint32_t)h->xid != (uint32_t)f.xid_base + (uint32_t)k)
        return RS_ORDER;
    return RS_OK;
}

/* a multi reply frame that passed results_check(): were its writes rolled back? */
RG_HD bool rs_rolled_back(const uint8_t *fr, const ResFraming &f, uint64_t k)
{
    int64_t ok, bad;
    rs_lens(f, k, &ok, &bad);
    const int32_t L = (int32_t)be32_at(fr);
    return L == bad && (L != ok || (int32_t)be32_at(fr + 20) == -1);
}

RG_HD bool rs_header_is(const uint8_t *q, int32_t type, uint8_t done, int32_t err)
{
    return (int32_t)be32_at(q) == type && q[4] == done && (int32_t)be32_at(q + 5) == err;
}

struct ResEntry {
    int32_t err;        /* the entry's own code (0, the failing code, -2 after it in a rolled-back multi) */
    int32_t version;    /* Stat.version of a setData that took effect, 0 for a create / replace that did, else -1 */
    uint8_t cls;        /* RS_DONE / RS_FAILED / RS_ABORTED */
    uint64_t at;        /* the byte of a fault */
};

/* A CreateResponse{P, path} at q against entry e's framed path */
RG_HD bool rs_echo_ok(const uint8_t *q, const ResFraming &f, uint64_t e)
{
    const unsigned long long o = f.path_off[e];
    const uint32_t P = (uint32_t)(f.path_off[e + 1] - o);
    if (be32_at(q) != P)
        return false;
    for (uint32_t t = 0; t < P; t++)
        if (q[4 + t] != f.path_bytes[o + t])
            return false;
    return true;
}

/* Entry e (of frame k, whose reply passed results_check() at fpos of the stream s) at its closed-form position: its
   results checked and its outcome.  `tol` is the code that still counts as done (NONODE for a delete, NODEEXISTS for a
   mkdirp create; 0 = none).  The entry that closes its multi frame also checks the closing header, and in a rolled-back
   frame that some ErrorResult is not 0.  Faults are reported at r->at; every read stays inside the frame. */
RG_HD uint32_t results_entry(const uint8_t *s, uint64_t fpos, const ResFraming &f, uint64_t k, uint64_t e, int32_t tol,
    ResEntry *r)
{
    const uint8_t *fr = s + fpos;
    const int32_t L = (int32_t)be32_at(fr), herr = (int32_t)be32_at(fr + 16);
    const uint64_t a = k * f.group, b = a + f.group < f.entries ? a + f.group : f.entries, i = e - a;
    r->err = 0;
    r->version = -1;
    r->cls = RS_DONE;
    r->at = fpos;
    if (herr != 0) {                                /* no body: every operation of the frame failed with err */
        r->err = herr;
        r->cls = herr == tol && tol != 0 ? RS_DONE : RS_FAILED;
        return RS_OK;
    }
    if (!f.multi) {
        if (f.op == 1u) {
            r->at = fpos + 20;
            if (!rs_echo_ok(fr + 20, f, e))
                return RS_PATH_ECHO;
            r->version = 0;
        } else if (f.op == 5u) {
            r->at = fpos + 20 + 52;
            if (be32_at(fr + 20 + 52) != (uint32_t)(f.data_off[e + 1] - f.data_off[e]))
                return RS_STAT_LEN;
            r->version = (int32_t)be32_at(fr + 20 + 32);
        }
        return RS_OK;
    }
    const uint32_t ops = rs_ops(f);
    const bool rolled = rs_rolled_back(fr, f, k);
    if (!rolled) {
        const bool echo = f.op == 1u || f.op == RS_REPLACE;     /* results that carry the path */
        uint64_t q = fpos + 20 + i * rs_fixed(f) + (echo ? f.path_off[e] - f.path_off[a] : 0ull);
        if (f.op == RS_REPLACE) {                   /* the delete (no result), then the create */
            r->at = q;
            if (!rs_header_is(s + q, 2, 0, 0))
                return RS_OP_TYPE;
            q += 9;
        }
        r->at = q;
        if (!rs_header_is(s + q, f.op == RS_REPLACE ? 1 : (int32_t)f.op, 0, 0))
            return RS_OP_TYPE;
        if (f.op == 1u || f.op == RS_REPLACE) {
            r->at = q + 9;
            if (!rs_echo_ok(s + q + 9, f, e))
                return RS_PATH_ECHO;
            r->version = 0;
        } else if (f.op == 5u) {
            r->at = q + 9 + 52;
            if (be32_at(s + q + 9 + 52) != (uint32_t)(f.data_off[e + 1] - f.data_off[e]))
                return RS_STAT_LEN;
            r->version = (int32_t)be32_at(s + q + 9 + 32);
        }
    } else {
        bool fails = false;
        int32_t own = 0, code_fail = 0;
        for (uint32_t t = 0; t < ops; t++) {
            const uint64_t j = i * ops + t, q = fpos + 20 + 13 * j;
            r->at = q;
            const int32_t c = (int32_t)be32_at(s + q + 5);
            if ((int32_t)be32_at(s + q) != -1 || s[q + 4] != 0)
                return RS_OP_TYPE;
            if ((int32_t)be32_at(s + q + 9) != c)
                return RS_ERR_RESULT;
            const int32_t prev = j ? (int32_t)be32_at(s + q - 13 + 9) : 0;
            if (prev != 0 && c != -2)               /* after the failing operation only -2 */
                return RS_ERR_SEQ;
            if (c != 0 && prev == 0) {
                fails = true;
                code_fail = c;
            }
            if (own == 0)
                own = c;
        }
        if (fails) {
            r->err = code_fail;
            r->cls = code_fail == tol && tol != 0 ? RS_DONE : RS_FAILED;
        } else {
            r->err = own;
            r->cls = RS_ABORTED;
        }
    }
    if (e + 1 == b) {                               /* the entry that closes the frame */
        const uint64_t q = fpos + 4 + (uint32_t)L - 9;
        r->at = q;
        if (!rs_header_is(s + q, -1, 1, -1))
            return RS_CLOSE;
        if (rolled && (int32_t)be32_at(s + q - 4) == 0)
            return RS_NO_FAILURE;
    }
    return RS_OK;
}

}  /* namespace regk */

#if defined(__CUDACC__)
#include "regk_kernels.cuh"

namespace regk {

/* counters[]: RQ_ERR .. RQ_STOP as regk_replies.cuh uses them, then these */
enum { RS_ENT_ERR = RQ_NCOUNTERS, RS_NDONE, RS_NFAILED, RS_NABORTED, RS_NCOUNTERS };

struct ResParams {
    RepParams r;                                /* the frame chain: r.n = frames */
    ResFraming f;
    uint64_t start;
    uint64_t n_eff;                             /* entries checked: those of the frames before the first frame fault */
    int32_t tol;
    unsigned long long *fpos;                   /* [frames] the reply's position */
    int32_t *ferr;                              /* [frames] its ReplyHeader.err */
    const unsigned long long *subject_in;       /* [entries] what entry e stands for; NULL = e itself */
    int32_t *err;                               /* [entries] */
    uint8_t *cls;
    int32_t *ver;
    unsigned long long *subject;
    unsigned long long *fault_at;               /* [entries] the byte of an entry's fault */
    uint32_t *tile_a, *tile_b;                  /* FAILED / ABORTED counts, two-level */
    unsigned long long *super_a, *super_b;
    unsigned long long *failed, *aborted;
};

/* ---- frames, cand: the plausible frame positions at or after start ---- */
__global__ void __launch_bounds__(RP_TILE) regk_results_cand_kernel(const ResParams rp)
{
    const RepParams &p = rp.r;
    __shared__ __align__(16) uint8_t s_win[RP_SPAN + 32];
    __shared__ uint32_t s_warp[WARPS];
    const uint64_t nblk = (p.len + 15u) / 16u;
    const uint64_t b0 = (uint64_t)blockIdx.x * RP_TILE, b = b0 + threadIdx.x;
    const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
    reinterpret_cast<uint4 *>(s_win)[threadIdx.x] = b < nblk ? rp_block(p.s, p.len, b) : zero;
    if (threadIdx.x < 2) {
        const uint64_t e = b0 + RP_TILE + threadIdx.x;
        reinterpret_cast<uint4 *>(s_win)[RP_TILE + threadIdx.x] = e < nblk ? rp_block(p.s, p.len, e) : zero;
    }
    __syncthreads();
    uint32_t mask = 0;
    if (b < nblk && 16ull * b + 16u > rp.start) {
        for (uint32_t f = 0; f < 16u; f++) {
            const uint64_t pos = 16ull * b + f;
            if (pos >= p.len)
                break;
            ResHead h;
            if (pos >= rp.start && results_head(s_win + 16u * threadIdx.x + f, p.len - pos, rp.f, &h) == RS_OK)
                mask |= 1u << f;
        }
    }
    uint32_t total;
    const uint32_t rank = block_scan<uint32_t>(s_warp, (uint32_t)__popc(mask), &total);
    if (b < nblk)
        p.word[b] = mask | rank << 16;
    if (threadIdx.x == 0)
        add_tile_total(p.tile_total, p.super_total, blockIdx.x, total);
}

/* ---- frames, chain: k of every reply frame, the check of k < frames, its position and err ---- */
__global__ void __launch_bounds__(RP_TILE) regk_results_chain_kernel(const ResParams rp)
{
    const RepParams &p = rp.r;
    __shared__ uint32_t s_warp[WARPS];
    __shared__ unsigned long long s_base;
    __shared__ uint32_t s_skip;
    if (threadIdx.x < 32) {
        const unsigned long long base = tile_base_from_totals(p.tile_total, p.super_total, blockIdx.x);
        if (threadIdx.x == 0) {
            s_base = base;
            s_skip = 0;
        }
    }
    const uint64_t c = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    const bool on = c < p.C && p.marked[c];
    const bool rep = rp_is_reply(p, c);
    uint32_t tot;
    const uint32_t r = block_scan<uint32_t>(s_warp, rep ? 1u : 0u, &tot);      /* its barriers publish s_base, s_skip */
    const uint64_t k = s_base + r;
    if (on && k < p.n) {
        if (!rep) {
            atomicAdd(&s_skip, 1u);
        } else {
            const unsigned long long pos = p.cand[c];
            ResHead h;
            const uint32_t code = results_check(p.s + pos, p.len - pos, rp.f, k, &h);
            rp.fpos[k] = pos;
            if (code != RS_OK) {
                atomicMin(p.counters + RQ_ERR, (unsigned long long)k << 8 | code);
            } else {
                rp.ferr[k] = h.err;
                if (k + 1 == p.n)
                    p.counters[RQ_CONSUMED] = pos + 4u + (uint32_t)h.len;
            }
        }
    }
    if (c + 1 == p.C)
        p.counters[RQ_NREP] = s_base + tot;
    __syncthreads();
    if (threadIdx.x == 0 && s_skip)
        atomicAdd(p.counters + RQ_SKIP, (unsigned long long)s_skip);
}

/* ---- entries: one thread per entry, its result at its closed-form position; FAILED / ABORTED counts per CTA ---- */
__global__ void __launch_bounds__(RP_TILE) regk_results_entry_kernel(const ResParams rp)
{
    __shared__ uint32_t s_cnt[3];
    if (threadIdx.x < 3)
        s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t e = (uint64_t)blockIdx.x * RP_TILE + threadIdx.x;
    uint32_t cls = 0xFFu;                           /* no entry */
    if (e < rp.n_eff) {
        const uint64_t k = e / rp.f.group;
        ResEntry r;
        const uint32_t code = results_entry(rp.r.s, rp.fpos[k], rp.f, k, e, rp.tol, &r);
        if (code != RS_OK) {
            rp.fault_at[e] = r.at;
            atomicMin(rp.r.counters + RS_ENT_ERR, (unsigned long long)e << 8 | code);
        }
        cls = r.cls;
        rp.err[e] = r.err;
        rp.cls[e] = r.cls;
        rp.ver[e] = r.version;
        rp.subject[e] = rp.subject_in ? rp.subject_in[e] : e;
        atomicAdd(&s_cnt[cls], 1u);
    }
    const uint32_t na = __popc(__ballot_sync(0xFFFFFFFFu, cls == RS_FAILED));
    const uint32_t nb = __popc(__ballot_sync(0xFFFFFFFFu, cls == RS_ABORTED));
    if ((threadIdx.x & 31u) == 0) {
        add_tile_total(rp.tile_a, rp.super_a, blockIdx.x, na);
        add_tile_total(rp.tile_b, rp.super_b, blockIdx.x, nb);
    }
    __syncthreads();
    if (threadIdx.x < 3 && s_cnt[threadIdx.x])
        atomicAdd(rp.r.counters + RS_NDONE + threadIdx.x, (unsigned long long)s_cnt[threadIdx.x]);
}

/* ---- where the frame chain stops short: results_head() there, into counters[RQ_M] (a refusal's message only) ---- */
__global__ void regk_results_head_kernel(const ResParams rp, unsigned long long pos)
{
    ResHead h;
    rp.r.counters[RQ_M] = results_head(rp.r.s + pos, rp.r.len - pos, rp.f, &h);
}

/* ---- lists: the FAILED and the ABORTED entries, ascending ---- */
__global__ void __launch_bounds__(RP_TILE) regk_results_list_kernel(const ResParams rp)
{
    __shared__ uint32_t s_warp[2][WARPS];
    __shared__ unsigned long long s_base[2];
    const uint32_t tile = blockIdx.x, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    if (threadIdx.x < 32) {
        const unsigned long long a = tile_base_from_totals(rp.tile_a, rp.super_a, tile);
        const unsigned long long b = tile_base_from_totals(rp.tile_b, rp.super_b, tile);
        if (threadIdx.x == 0) {
            s_base[0] = a;
            s_base[1] = b;
        }
    }
    const uint64_t e = (uint64_t)tile * RP_TILE + threadIdx.x;
    const uint32_t c = e < rp.n_eff ? rp.cls[e] : (uint32_t)RS_DONE;
    const uint32_t ba = __ballot_sync(0xFFFFFFFFu, c == RS_FAILED), bb = __ballot_sync(0xFFFFFFFFu, c == RS_ABORTED);
    if (lane == 0) {
        s_warp[0][warp] = __popc(ba);
        s_warp[1][warp] = __popc(bb);
    }
    __syncthreads();
    uint32_t ra = __popc(ba & ((1u << lane) - 1u)), rb = __popc(bb & ((1u << lane) - 1u));
    #pragma unroll
    for (uint32_t w = 0; w < WARPS; w++) {
        if (w < warp) {
            ra += s_warp[0][w];
            rb += s_warp[1][w];
        }
    }
    if (c == RS_FAILED)
        rp.failed[s_base[0] + ra] = e;
    else if (c == RS_ABORTED)
        rp.aborted[s_base[1] + rb] = e;
}

}  /* namespace regk */
#endif /* __CUDACC__ */
#endif /* REGK_RESULTS_CUH */
