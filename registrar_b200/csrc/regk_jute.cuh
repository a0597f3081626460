/*
 * regk_jute.cuh — ZooKeeper wire framing of a finished batch (SURVEY.md §8(f).3).
 *
 * Reference call site: lib/register.js:156-159  zk.create(n, _obj, {flags: ['ephemeral_plus']}, cb)  - what zkplus
 * (package.json:20, NOT in the reference tree) finally writes to the socket is one jute-serialised request per node.
 * PARITY UNPINNED: neither zkplus nor a ZooKeeper client is available here, so the layout below is restated from
 * the published ZooKeeper protocol (zookeeper.jute: RequestHeader, CreateRequest, ACL, Id; all integers big
 * endian) and checked only against an independent Python restatement of the same definition (oracle/pyoracle.py).
 *
 *   int   len                      bytes that follow (frame length - 4)
 *   int   xid                      RequestHeader.xid        xid_base + record index
 *   int   type = 1                 RequestHeader.type       OpCode.create
 *   int   path length, path bytes  CreateRequest.path       (ustring)
 *   int   data length, data bytes  CreateRequest.data       (buffer)  the JSON payload
 *   int   1                        CreateRequest.acl        vector<ACL> with one element: OPEN_ACL_UNSAFE
 *   int   31                         ACL.perms              ZooDefs.Perms.ALL
 *   int   5, "world"                 ACL.id.scheme
 *   int   6, "anyone"                ACL.id.id
 *   int   flags                    CreateRequest.flags      1 = EPHEMERAL (what 'ephemeral_plus' creates; zkplus
 *                                                           re-creates the node after a session loss by itself)
 * A frame is P + J + 51 bytes, so frame_off[i] = path_off[i] + json_off[i] + 51 i: closed form, no scan.
 *
 * Kernel: pure concatenation of two packed streams plus 51 framing bytes per record - HBM-bound byte shuffling with
 * nothing to compute, so it is written OUTPUT-STATIONARY: one CTA per tile of JUTE_TILE records stages the tile's
 * slices of both streams in shared memory (two cp.async.bulk copies), builds the 20 variable framing bytes of every
 * record (four big-endian header words + the data length) and the constant 31-byte trailer there as well, and then
 * every thread produces whole 16-byte blocks of the OUTPUT: it finds the record its block starts in (binary search
 * over the tile's closed-form frame offsets), walks the segments that overlap the block (header | path | data
 * length | data | trailer - all plain byte ranges of shared memory by now), fetches each with one unaligned 16-byte
 * load positioned so that every source byte lands on its destination lane, merges under a byte mask from a small
 * table, and stores the block with one coalesced 128-bit store.  No lane ever idles on a short record, nothing is
 * written twice, and the only byte-sized stores are the two ragged blocks at the ends of a tile.  (The first
 * version copied byte by byte, a warp per record: 3.83 ms per 10 M records = 0.18 of the HBM peak; this one:
 * see DESIGN.md §4.)  Tiles whose slices exceed the staging budget fall back to the byte-wise path.
 */
#ifndef REGK_JUTE_CUH
#define REGK_JUTE_CUH

#include "regk_kernels.cuh"

namespace regk {

constexpr uint32_t JUTE_TILE = 64;              /* records per CTA */
constexpr uint32_t JUTE_THREADS = 128;
constexpr uint32_t JUTE_SLOT = 32;              /* per-record framing slot in shared memory: the head RIGHT-aligned so that it
                                                   ends at byte 28, the data length in bytes 28..31 */
constexpr uint32_t JUTE_FRAME_HEAD = 12;        /* len, xid, type: once per frame */
constexpr uint32_t JUTE_MULTI_HEAD = 9;         /* MultiHeader {int type; boolean done; int err}: in front of every operation */
constexpr uint32_t JUTE_TAIL_MAX = 31;          /* create: acl count, perms, scheme, id, flags */
enum : uint32_t { JUTE_OP_CREATE = 1, JUTE_OP_DELETE = 2, JUTE_OP_SETDATA = 5, JUTE_OP_MULTI = 14 };

struct JuteParams {
    uint64_t n;
    const uint8_t *path_bytes;
    const unsigned long long *path_off;         /* [n+1] */
    const uint8_t *json_bytes;                  /* NULL when the operation carries no data (delete) */
    const unsigned long long *json_off;         /* [n+1] */
    uint8_t *out_bytes;
    unsigned long long *out_off;                /* [frames+1] */
    uint64_t out_capacity;
    int32_t xid_base;
    uint32_t op;                                /* JUTE_OP_CREATE / DELETE / SETDATA */
    uint32_t mid;                               /* 4: a data buffer follows the path (its length word), 0: none */
    uint32_t tail_len;                          /* bytes behind the data: create 31 (acl + flags), delete / setData 4 (version) */
    uint32_t tail[12];                          /* those bytes, then the 9 bytes that close a multi transaction */
    uint32_t group;                             /* operations per frame: 1 unless `multi` */
    uint32_t multi;                             /* 1: frames are multi transactions of `group` operations */
    uint32_t per_rec;                           /* framing bytes every record carries: (multi ? 9 : 0) + 4 + mid + tail_len */
    uint32_t path_cap, json_cap;                /* shared-memory budgets of the staged slices (bytes, multiples of 16) */
    uint64_t path_limit, json_limit;            /* bytes readable behind path_bytes / json_bytes (whole 16-byte blocks are fetched) */
    DevStatus *status;
};

__device__ __forceinline__ uint32_t bswap32(uint32_t v)
{
    return __byte_perm(v, 0u, 0x0123);
}

/*
 * The framing slot of one record (8 little-endian words = 32 bytes as they go on the wire):
 *   single request   bytes 12..27  len | xid | op | path length                      28..31 data length
 *   multi operation  bytes  3..27  len | xid | 14 | op | done = 0 | err = -1 | path length   (a record that does not
 *                    open a frame uses bytes 15..27 only)
 * `frame_len` is only read for a record that opens a frame.
 */
template <bool MULTI>
__device__ __forceinline__ void jute_slot(const JuteParams &p, uint32_t xid, uint32_t frame_len, uint32_t P, uint32_t J,
    uint32_t (&h)[8])
{
    if (!MULTI) {
        h[0] = h[1] = h[2] = 0u;
        h[3] = bswap32(frame_len);
        h[4] = bswap32(xid);
        h[5] = bswap32(p.op);
    } else {
        const uint32_t x0 = bswap32(frame_len), x1 = bswap32(xid), x2 = bswap32(JUTE_OP_MULTI), x3 = bswap32(p.op);
        h[0] = x0 << 24;
        h[1] = (x0 >> 8) | (x1 << 24);
        h[2] = (x1 >> 8) | (x2 << 24);
        h[3] = (x2 >> 8) | (x3 << 24);
        h[4] = x3 >> 8;                                         /* byte 19: done = false */
        h[5] = 0xFFFFFFFFu;                                     /* err = -1 */
    }
    h[6] = bswap32(P);
    h[7] = bswap32(J);
}

/* byte masks of a 16-byte block: JUTE_GE[d] = bytes at index >= d, JUTE_LT[e] = bytes at index < e (d, e in 0..16) */
__device__ __forceinline__ uint4 mask_ge(uint32_t d)
{
    uint4 m;
    m.x = d >= 4u ? 0u : 0xFFFFFFFFu << (8u * d);
    m.y = d >= 8u ? 0u : d <= 4u ? 0xFFFFFFFFu : 0xFFFFFFFFu << (8u * (d - 4u));
    m.z = d >= 12u ? 0u : d <= 8u ? 0xFFFFFFFFu : 0xFFFFFFFFu << (8u * (d - 8u));
    m.w = d >= 16u ? 0u : d <= 12u ? 0xFFFFFFFFu : 0xFFFFFFFFu << (8u * (d - 12u));
    return m;
}

template <bool MULTI, bool DATA>
__global__ void __launch_bounds__(JUTE_THREADS) regk_jute_kernel(const JuteParams p)
{
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ uint32_t s_foff[JUTE_TILE + 1], s_poff[JUTE_TILE + 1], s_joff[JUTE_TILE + 1];
    __shared__ uint32_t s_nlist;
    __shared__ uint4 s_rec[JUTE_TILE];          /* {frame offset, path source | head bytes << 24, payload source | tail bytes << 24, P | J << 16} */
    const uint32_t t = threadIdx.x;
    const uint64_t r0 = (uint64_t)blockIdx.x * JUTE_TILE;
    const uint32_t nrec = (uint32_t)min((uint64_t)JUTE_TILE, p.n - r0);
    const uint32_t mid = DATA ? 4u : 0u, g = MULTI ? p.group : 1u;
    /* tile extents in the three streams (uniform loads) */
    const unsigned long long P0 = p.path_off[r0], P1 = p.path_off[r0 + nrec];
    const unsigned long long J0 = DATA ? p.json_off[r0] : 0ull, J1 = DATA ? p.json_off[r0 + nrec] : 0ull;
    const uint64_t q0 = MULTI ? r0 / g : r0;                    /* frames opened before the one r0 lies in */
    const uint32_t m0 = (uint32_t)(r0 - q0 * g);                /* r0's position inside its frame */
    /* framing bytes in front of record r0 + d (d <= 64; r0 + d <= n): every record's own, 12 per frame opened, 9 per
       multi frame closed */
    auto fixed_before = [&](uint32_t d) -> unsigned long long {
        if (!MULTI)
            return (unsigned long long)(p.per_rec + JUTE_FRAME_HEAD) * (r0 + d);
        const uint32_t md = m0 + d, fl = md / g, ce = (md + g - 1u) / g;
        return (unsigned long long)p.per_rec * (r0 + d) + (unsigned long long)JUTE_FRAME_HEAD * (q0 + ce) +
            (unsigned long long)JUTE_MULTI_HEAD * (q0 + (r0 + d == p.n ? ce : fl));
    };
    const unsigned long long f0 = P0 + J0 + fixed_before(0), f1 = P1 + J1 + fixed_before(nrec);
    const uint32_t total = (uint32_t)(f1 - f0);
    const bool room = f1 <= p.out_capacity;
    /* dynamic shared memory (byte space shared by every segment source, 16 bytes of slack around each region):
       [mask tables 2 x 17 x 16][framing slots: 32 bytes per record][tail 48][path slice][payload slice] */
    uint4 *s_ge = reinterpret_cast<uint4 *>(smem);
    uint4 *s_lt = s_ge + 17;
    const uint32_t HDR = 34u * 16u + 16u;                       /* byte offset of the per-record framing */
    const uint32_t TAIL = HDR + JUTE_TILE * JUTE_SLOT + 16u;
    const uint32_t PATH = TAIL + 48u + 16u;
    const uint32_t plead = (uint32_t)P0 & 15u, jlead = (uint32_t)J0 & 15u;
    const uint32_t np = (plead + (uint32_t)(P1 - P0) + 15u) & ~15u, nj = DATA ? (jlead + (uint32_t)(J1 - J0) + 15u) & ~15u : 0u;
    const uint32_t JSON = PATH + p.path_cap + 16u;
    const bool fits = room && np <= p.path_cap && (P0 & ~15ull) + np <= p.path_limit &&
        (!DATA || (nj <= p.json_cap && (J0 & ~15ull) + nj <= p.json_limit));
    if (t == 0) {
        mbar_init(&s_bar, 1);
        if (fits) {
            mbar_expect_tx(&s_bar, np + nj);
            if (np)
                bulk_g2s(smem + PATH, p.path_bytes + (P0 & ~15ull), np, &s_bar);
            if (nj)
                bulk_g2s(smem + JSON, p.json_bytes + (J0 & ~15ull), nj, &s_bar);
        }
    }
    /* this thread's record: where it sits in its frame, what framing it carries */
    const uint32_t mt = m0 + t;                                 /* t <= 64: no overflow concerns */
    const uint32_t fq = MULTI ? mt / g : t, fm = MULTI ? mt - fq * g : 0u;
    const bool first = fm == 0u;
    const bool last = !MULTI || fm == g - 1u || r0 + t + 1u == p.n;
    unsigned long long fo = 0;
    if (t <= nrec) {
        const unsigned long long po = p.path_off[r0 + t], jo = DATA ? p.json_off[r0 + t] : 0ull;
        fo = po + jo + fixed_before(t);
        s_poff[t] = (uint32_t)(po - P0);
        s_joff[t] = (uint32_t)(jo - J0);
        s_foff[t] = (uint32_t)(fo - f0);
        if (first && (t < nrec || r0 + nrec == p.n))
            p.out_off[MULTI ? q0 + fq : r0 + t] = fo;           /* the closing entry: r0 + t == n */
        else if (MULTI && t == nrec && r0 + nrec == p.n)
            p.out_off[q0 + fq + 1u] = fo;                       /* n is not a multiple of the group size */
    }
    if (t < 17) {
        s_ge[t] = mask_ge(t);
        const uint4 gm = mask_ge(t);
        s_lt[t] = make_uint4(~gm.x, ~gm.y, ~gm.z, ~gm.w);
    }
    if (t >= 32 && t < 44)                                      /* the tail: constant bytes, then the multi close */
        reinterpret_cast<uint32_t *>(smem + TAIL)[t - 32u] = p.tail[t - 32u];
    if (!room) {
        if (t == 0)
            atomicOr(&p.status->overflow, 1u);
        return;
    }
    const uint32_t hb = (first ? JUTE_FRAME_HEAD : 0u) + (MULTI ? JUTE_MULTI_HEAD : 0u) + 4u;
    const uint32_t tb = p.tail_len + (MULTI && last ? JUTE_MULTI_HEAD : 0u);
    /* the record's framing slot: lengths, xid, and - for the record that opens a multi frame - the frame's length,
       the distance to the record that opens the next one */
    auto make_slot = [&](uint32_t (&h)[8]) {
        const uint32_t P = (uint32_t)(p.path_off[r0 + t + 1] - p.path_off[r0 + t]);
        const uint32_t J = DATA ? (uint32_t)(p.json_off[r0 + t + 1] - p.json_off[r0 + t]) : 0u;
        uint32_t frame_len = P + J + hb + mid + tb - 4u;
        if (MULTI && first) {                                   /* the whole transaction: its operations, head and close */
            const uint64_t i = r0 + t, e = min(i + (uint64_t)g, p.n);
            frame_len = (uint32_t)(p.path_off[e] - p.path_off[i]) + (DATA ? (uint32_t)(p.json_off[e] - p.json_off[i]) : 0u) +
                p.per_rec * (uint32_t)(e - i) + JUTE_FRAME_HEAD + JUTE_MULTI_HEAD - 4u;
        }
        jute_slot<MULTI>(p, (uint32_t)p.xid_base + (uint32_t)(MULTI ? q0 + fq : r0 + t), frame_len, P, J, h);
    };
    if (!fits) {
        /* byte-wise fallback: a thread per record, straight to global memory */
        if (t < nrec) {
            uint32_t h[8];
            make_slot(h);
            uint8_t *gp = p.out_bytes + fo;
            const uint8_t *hbytes = reinterpret_cast<const uint8_t *>(h), *tbytes = reinterpret_cast<const uint8_t *>(p.tail);
            const uint32_t P = bswap32(h[6]), J = bswap32(h[7]);
            const uint8_t *ps = p.path_bytes + p.path_off[r0 + t];
            for (uint32_t k = 0; k < hb; k++)
                *gp++ = hbytes[28u - hb + k];
            for (uint32_t k = 0; k < P; k++)
                *gp++ = ps[k];
            if (DATA) {
                const uint8_t *js = p.json_bytes + p.json_off[r0 + t];
                for (uint32_t k = 0; k < 4u; k++)
                    *gp++ = hbytes[28u + k];
                for (uint32_t k = 0; k < J; k++)
                    *gp++ = js[k];
            }
            for (uint32_t k = 0; k < tb; k++)
                *gp++ = tbytes[k];
        }
        return;
    }
    __syncthreads();                                            /* offsets, masks, tail, mbarrier init */
    if (t < nrec) {
        uint32_t h[8];
        make_slot(h);
        uint4 *slot = reinterpret_cast<uint4 *>(smem + HDR + JUTE_SLOT * t);
        slot[0] = make_uint4(h[0], h[1], h[2], h[3]);
        slot[1] = make_uint4(h[4], h[5], h[6], h[7]);
        s_rec[t] = make_uint4(s_foff[t], (PATH + plead + s_poff[t]) | (MULTI ? hb << 24 : 0u),
            (JSON + jlead + s_joff[t]) | (MULTI ? tb << 24 : 0u), bswap32(h[6]) | (bswap32(h[7]) << 16));
    }
    const unsigned long long a0 = f0 & ~15ull;
    const uint32_t lead = (uint32_t)(f0 - a0);
    const uint32_t nblk = (lead + total + 15u) >> 4;
    /* which record does output block b start in?  every record marks the blocks whose first byte (for block 0:
       the tile's first byte) lies inside its frame - about 16 byte-sized stores per record instead of a binary
       search per block */
    uint8_t *s_owner = smem + JSON + p.json_cap + 48u;
    if (t < nrec) {
        const uint32_t fa = s_foff[t] + lead, fb = s_foff[t + 1] + lead;    /* frame range in block coordinates (bytes) */
        uint32_t b = t == 0 ? 0u : (fa + 15u) >> 4;
        for (; 16u * b < fb && b < nblk; b++)
            s_owner[b] = (uint8_t)t;
    }
    mbar_wait(&s_bar, 0);
    __syncthreads();
    const uint32_t *sw = reinterpret_cast<const uint32_t *>(smem);
    /* Phase 1: blocks that lie entirely inside ONE path or payload segment (about 70 % of them) are a straight
       realigned copy - no masks, no segment walk, every lane busy; the others are only listed.  Phase 2 takes the
       list, compacted, through the general walk - so the lanes of a warp no longer wait for the one block that
       straddles three segments. */
    uint16_t *s_list = reinterpret_cast<uint16_t *>(s_owner + ((nblk + 15u) & ~15u));
    if (t == 0)
        s_nlist = 0;
    __syncthreads();
    for (uint32_t b = t; b < nblk; b += JUTE_THREADS) {
        const int32_t bstart = (int32_t)(16u * b) - (int32_t)lead;
        const uint32_t i = s_owner[b];
        const uint4 rc = s_rec[i];
        const uint32_t fo_b = (uint32_t)bstart - rc.x;          /* meaningful when bstart >= 0 */
        const uint32_t P = rc.w & 0xFFFFu, J = rc.w >> 16;
        const uint32_t ph = MULTI ? rc.y >> 24 : JUTE_FRAME_HEAD + 4u;         /* head bytes of record i */
        const bool whole = bstart >= 0 && (uint32_t)bstart + 16u <= total;
        const bool in_path = fo_b >= ph && fo_b + 16u <= ph + P;
        const bool in_data = fo_b >= ph + P + mid && fo_b + 16u <= ph + P + mid + J;
        if (whole && (in_path || in_data)) {
            const uint32_t ys = MULTI ? rc.y & 0xFFFFFFu : rc.y, zs = MULTI ? rc.z & 0xFFFFFFu : rc.z;
            const uint32_t src = in_path ? ys + (fo_b - ph) : zs + (fo_b - ph - P - mid);
            uint32_t v[4];
            load16(sw, src, v);
            stg_v4(p.out_bytes + a0 + 16ull * b, make_uint4(v[0], v[1], v[2], v[3]));
        } else {
            s_list[atomicAdd(&s_nlist, 1u)] = (uint16_t)b;
        }
    }
    __syncthreads();
    const uint32_t nlist = s_nlist;
    for (uint32_t li = t; li < nlist; li += JUTE_THREADS) {
        const uint32_t b = s_list[li];
        const int32_t bstart = (int32_t)(16u * b) - (int32_t)lead;     /* tile-relative frame byte of the block's byte 0 */
        uint32_t pos = bstart < 0 ? 0u : (uint32_t)bstart;
        const uint32_t end = min((uint32_t)(bstart + 16), total);
        uint32_t i = s_owner[b];                                /* the record the block starts in */
        uint32_t acc[4] = {0u, 0u, 0u, 0u};
        while (pos < end) {
            const uint4 rc = s_rec[i];                          /* one 128-bit load per step */
            const uint32_t fo_b = pos - rc.x;
            const uint32_t P = rc.w & 0xFFFFu, J = rc.w >> 16;
            const uint32_t ph = MULTI ? rc.y >> 24 : JUTE_FRAME_HEAD + 4u, pt = MULTI ? rc.z >> 24 : p.tail_len;
            const uint32_t ys = MULTI ? rc.y & 0xFFFFFFu : rc.y, zs = MULTI ? rc.z & 0xFFFFFFu : rc.z;
            uint32_t src, seg_end;
            if (fo_b < ph) {
                src = HDR + JUTE_SLOT * i + 28u - ph + fo_b;
                seg_end = ph;
            } else if (fo_b < ph + P) {
                src = ys + (fo_b - ph);
                seg_end = ph + P;
            } else if (fo_b < ph + P + mid) {
                src = HDR + JUTE_SLOT * i + 28u + (fo_b - ph - P);
                seg_end = ph + P + mid;
            } else if (fo_b < ph + P + mid + J) {
                src = zs + (fo_b - ph - P - mid);
                seg_end = ph + P + mid + J;
            } else {
                src = TAIL + (fo_b - ph - P - mid - J);
                seg_end = ph + P + mid + J + pt;
            }
            const uint32_t n = min(seg_end - fo_b, end - pos);
            const uint32_t d = (uint32_t)((int32_t)pos - bstart);       /* destination byte inside the block */
            uint32_t v[4];
            load16(sw, src - d, v);                             /* source byte k lands on lane byte d + k */
            const uint4 mg = s_ge[d], ml = s_lt[d + n];
            acc[0] |= v[0] & mg.x & ml.x;
            acc[1] |= v[1] & mg.y & ml.y;
            acc[2] |= v[2] & mg.z & ml.z;
            acc[3] |= v[3] & mg.w & ml.w;
            pos += n;
            if (fo_b + n == ph + P + mid + J + pt)
                i++;
        }
        uint8_t *gp = p.out_bytes + a0 + 16ull * b;
        if (bstart >= 0 && (uint32_t)bstart + 16u <= total) {
            stg_v4(gp, make_uint4(acc[0], acc[1], acc[2], acc[3]));
        } else {                                                /* the tile's ragged first / last block: its own bytes only */
            const uint32_t d0 = bstart < 0 ? (uint32_t)(-bstart) : 0u, d1 = end - (uint32_t)max(bstart, 0) + d0;
            for (uint32_t k = d0; k < d1; k++)
                gp[k] = (uint8_t)(acc[k >> 2] >> (8u * (k & 3u)));
        }
    }
}

/*
 * Versioned and paired framing: regk_reconcile_requests after regk_reconcile_owned (REGK_ZK_VERSION_OBSERVED on delete /
 * setData, and REGK_ZK_REPLACE).  The same output-stationary scheme as regk_jute_kernel, with the framing of every
 * entry built in a slot of its own instead of a constant tail, and the path segment emitted twice for a replace.  An
 * entry is seven segments
 *     F0 | path | F1 | path again | F2 | data | F3
 * F0..F3 are framing bytes, contiguous in the entry's 96-byte shared-memory slot (F0 right-aligned to end at byte 32,
 * F1, F2, F3 behind it), so a framing byte's source is slot + 32 - f0 + (its offset in the entry - the stream bytes
 * in front of it):
 *   delete           F0 = head | path length                                          F3 = version [| close]
 *   setData          F0 = head | path length               F2 = data length           F3 = version [| close]
 *   replace (PAIR)   F0 = head | MultiHeader{2} | path length   F1 = version | MultiHeader{1} | path length
 *                    F2 = data length                      F3 = acl | zk_flags [| close]
 * head = len | xid | op for a single request; in a multi frame len | xid | 14 | MultiHeader{op, false, -1} for the entry
 * that opens it and MultiHeader{op, false, -1} for the others; close = MultiHeader{-1, true, -1}.  A replace entry is
 * 65 + 2 P + J bytes, so entry r starts at (1 + PAIR) path_off[r] + json_off[r] + per_rec r + 12 per frame opened before
 * it + 9 per frame closed before it: closed form, as in regk_jute_kernel.
 */
constexpr uint32_t JUTE_ESLOT = 96;             /* framing slot of one entry: at most 25 + 17 + 4 + 40 bytes from byte 7 */

struct JuteEntryParams {
    uint64_t n;
    const uint8_t *path_bytes;
    const unsigned long long *path_off;         /* [n+1] */
    const uint8_t *json_bytes;                  /* NULL without data (delete) */
    const unsigned long long *json_off;
    const int32_t *version;                     /* [n] the expected version of each entry, or NULL: version_const */
    int32_t version_const;
    uint32_t op;                                /* JUTE_OP_DELETE / SETDATA; PAIR: JUTE_OP_DELETE, then a create */
    uint32_t zk_flags;                          /* PAIR: CreateMode of the creates */
    uint32_t group;                             /* entries per frame: 1 unless MULTI */
    uint32_t per_rec;                           /* framing bytes every entry carries, frame head and close excluded */
    int32_t xid_base;
    uint8_t *out_bytes;
    unsigned long long *out_off;                /* [frames+1] */
    uint64_t out_capacity;
    uint32_t path_cap, json_cap;
    uint64_t path_limit, json_limit;
    DevStatus *status;
};

__constant__ uint8_t JUTE_OPEN_ACL[27] = {0, 0, 0, 1, 0, 0, 0, 31, 0, 0, 0, 5, 'w', 'o', 'r', 'l', 'd',
                                          0, 0, 0, 6, 'a', 'n', 'y', 'o', 'n', 'e'};

__device__ __forceinline__ void put_be32(uint8_t *s, uint32_t v)
{
    s[0] = (uint8_t)(v >> 24);
    s[1] = (uint8_t)(v >> 16);
    s[2] = (uint8_t)(v >> 8);
    s[3] = (uint8_t)v;
}

__device__ __forceinline__ void put_multi_header(uint8_t *s, uint32_t op, uint32_t done)
{
    put_be32(s, op);
    s[4] = (uint8_t)done;
    put_be32(s + 5, 0xFFFFFFFFu);
}

template <bool MULTI, bool DATA, bool PAIR>
__global__ void __launch_bounds__(JUTE_THREADS) regk_jute_entry_kernel(const JuteEntryParams p)
{
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ __align__(8) uint64_t s_bar;
    __shared__ uint32_t s_foff[JUTE_TILE + 1], s_poff[JUTE_TILE + 1], s_joff[JUTE_TILE + 1];
    __shared__ uint32_t s_nlist;
    __shared__ uint4 s_rec[JUTE_TILE];          /* {frame offset, path source | f0 << 24, payload source | f3 << 24, P | J << 16} */
    constexpr uint32_t PM = PAIR ? 2u : 1u;     /* times the path is emitted */
    constexpr uint32_t F1 = PAIR ? 17u : 0u, F2 = DATA ? 4u : 0u, F3 = PAIR ? 31u : 4u;
    const uint32_t t = threadIdx.x;
    const uint64_t r0 = (uint64_t)blockIdx.x * JUTE_TILE;
    const uint32_t nrec = (uint32_t)min((uint64_t)JUTE_TILE, p.n - r0);
    const uint32_t g = MULTI ? p.group : 1u;
    const unsigned long long P0 = p.path_off[r0], P1 = p.path_off[r0 + nrec];
    const unsigned long long J0 = DATA ? p.json_off[r0] : 0ull, J1 = DATA ? p.json_off[r0 + nrec] : 0ull;
    const uint64_t q0 = MULTI ? r0 / g : r0;
    const uint32_t m0 = (uint32_t)(r0 - q0 * g);
    auto fixed_before = [&](uint32_t d) -> unsigned long long {
        if (!MULTI)
            return (unsigned long long)(p.per_rec + JUTE_FRAME_HEAD) * (r0 + d);
        const uint32_t md = m0 + d, fl = md / g, ce = (md + g - 1u) / g;
        return (unsigned long long)p.per_rec * (r0 + d) + (unsigned long long)JUTE_FRAME_HEAD * (q0 + ce) +
            (unsigned long long)JUTE_MULTI_HEAD * (q0 + (r0 + d == p.n ? ce : fl));
    };
    const unsigned long long f0 = PM * P0 + J0 + fixed_before(0), f1 = PM * P1 + J1 + fixed_before(nrec);
    const uint32_t total = (uint32_t)(f1 - f0);
    const bool room = f1 <= p.out_capacity;
    /* dynamic shared memory: [mask tables 2 x 17 x 16][framing slots: 96 bytes per entry][path slice][payload slice] */
    uint4 *s_ge = reinterpret_cast<uint4 *>(smem);
    uint4 *s_lt = s_ge + 17;
    const uint32_t HDR = 34u * 16u + 16u;
    const uint32_t PATH = HDR + JUTE_TILE * JUTE_ESLOT + 16u;
    const uint32_t plead = (uint32_t)P0 & 15u, jlead = (uint32_t)J0 & 15u;
    const uint32_t np = (plead + (uint32_t)(P1 - P0) + 15u) & ~15u, nj = DATA ? (jlead + (uint32_t)(J1 - J0) + 15u) & ~15u : 0u;
    const uint32_t JSON = PATH + p.path_cap + 16u;
    const bool fits = room && np <= p.path_cap && (P0 & ~15ull) + np <= p.path_limit &&
        (!DATA || (nj <= p.json_cap && (J0 & ~15ull) + nj <= p.json_limit));
    if (t == 0) {
        mbar_init(&s_bar, 1);
        if (fits) {
            mbar_expect_tx(&s_bar, np + nj);
            if (np)
                bulk_g2s(smem + PATH, p.path_bytes + (P0 & ~15ull), np, &s_bar);
            if (nj)
                bulk_g2s(smem + JSON, p.json_bytes + (J0 & ~15ull), nj, &s_bar);
        }
    }
    const uint32_t mt = m0 + t;
    const uint32_t fq = MULTI ? mt / g : t, fm = MULTI ? mt - fq * g : 0u;
    const bool first = fm == 0u;
    const bool last = !MULTI || fm == g - 1u || r0 + t + 1u == p.n;
    unsigned long long fo = 0;
    if (t <= nrec) {
        const unsigned long long po = p.path_off[r0 + t], jo = DATA ? p.json_off[r0 + t] : 0ull;
        fo = PM * po + jo + fixed_before(t);
        s_poff[t] = (uint32_t)(po - P0);
        s_joff[t] = (uint32_t)(jo - J0);
        s_foff[t] = (uint32_t)(fo - f0);
        if (first && (t < nrec || r0 + nrec == p.n))
            p.out_off[MULTI ? q0 + fq : r0 + t] = fo;
        else if (MULTI && t == nrec && r0 + nrec == p.n)
            p.out_off[q0 + fq + 1u] = fo;
    }
    if (t < 17) {
        s_ge[t] = mask_ge(t);
        const uint4 gm = mask_ge(t);
        s_lt[t] = make_uint4(~gm.x, ~gm.y, ~gm.z, ~gm.w);
    }
    if (!room) {
        if (t == 0)
            atomicOr(&p.status->overflow, 1u);
        return;
    }
    const uint32_t fh = (first ? JUTE_FRAME_HEAD : 0u) + (MULTI ? JUTE_MULTI_HEAD : 0u) + 4u;     /* f0 */
    const uint32_t ft = F3 + (MULTI && last ? JUTE_MULTI_HEAD : 0u);                               /* f3 */
    uint8_t *slot = smem + HDR + JUTE_ESLOT * t;
    uint32_t P = 0, J = 0;
    /* this entry's framing bytes into its slot */
    auto make_slot = [&]() {
        const uint64_t i = r0 + t;
        P = (uint32_t)(p.path_off[i + 1] - p.path_off[i]);
        J = DATA ? (uint32_t)(p.json_off[i + 1] - p.json_off[i]) : 0u;
        uint32_t frame_len = PM * P + J + fh + F1 + F2 + ft - 4u;
        if (MULTI && first) {
            const uint64_t e = min(i + (uint64_t)g, p.n);
            frame_len = PM * (uint32_t)(p.path_off[e] - p.path_off[i]) + (DATA ? (uint32_t)(p.json_off[e] - p.json_off[i]) : 0u) +
                p.per_rec * (uint32_t)(e - i) + JUTE_FRAME_HEAD + JUTE_MULTI_HEAD - 4u;
        }
        const uint32_t v = (uint32_t)(p.version ? p.version[i] : p.version_const);
        uint8_t *s = slot + 32u - fh;
        if (first) {
            put_be32(s, frame_len);
            put_be32(s + 4, (uint32_t)p.xid_base + (uint32_t)(MULTI ? q0 + fq : i));
            put_be32(s + 8, MULTI ? JUTE_OP_MULTI : p.op);
            s += JUTE_FRAME_HEAD;
        }
        if (MULTI) {
            put_multi_header(s, p.op, 0u);
            s += JUTE_MULTI_HEAD;
        }
        put_be32(s, P);
        s = slot + 32u;
        if (PAIR) {
            put_be32(s, v);
            put_multi_header(s + 4, JUTE_OP_CREATE, 0u);
            put_be32(s + 13, P);
            s += F1;
        }
        if (DATA) {
            put_be32(s, J);
            s += F2;
        }
        if (PAIR) {
            for (uint32_t k = 0; k < 27u; k++)
                s[k] = JUTE_OPEN_ACL[k];
            put_be32(s + 27, p.zk_flags);
        } else {
            put_be32(s, v);
        }
        s += F3;
        if (MULTI && last)
            put_multi_header(s, 0xFFFFFFFFu, 1u);
    };
    if (!fits) {
        /* byte-wise fallback: a thread per entry, its slot, then straight to global memory */
        if (t < nrec) {
            make_slot();
            uint8_t *gp = p.out_bytes + fo;
            const uint8_t *fs = slot + 32u - fh, *ps = p.path_bytes + p.path_off[r0 + t];
            for (uint32_t k = 0; k < fh; k++)
                *gp++ = *fs++;
            for (uint32_t k = 0; k < P; k++)
                *gp++ = ps[k];
            if constexpr (PAIR) {
                for (uint32_t k = 0; k < F1; k++)
                    *gp++ = *fs++;
                for (uint32_t k = 0; k < P; k++)
                    *gp++ = ps[k];
            }
            if constexpr (DATA) {
                const uint8_t *js = p.json_bytes + p.json_off[r0 + t];
                for (uint32_t k = 0; k < F2; k++)
                    *gp++ = *fs++;
                for (uint32_t k = 0; k < J; k++)
                    *gp++ = js[k];
            }
            for (uint32_t k = 0; k < ft; k++)
                *gp++ = *fs++;
        }
        return;
    }
    __syncthreads();                                            /* offsets, masks, mbarrier init */
    if (t < nrec) {
        make_slot();
        s_rec[t] = make_uint4(s_foff[t], (PATH + plead + s_poff[t]) | (fh << 24), (JSON + jlead + s_joff[t]) | (ft << 24),
                              P | (J << 16));
    }
    const unsigned long long a0 = f0 & ~15ull;
    const uint32_t lead = (uint32_t)(f0 - a0);
    const uint32_t nblk = (lead + total + 15u) >> 4;
    uint8_t *s_owner = smem + JSON + p.json_cap + 48u;
    if (t < nrec) {
        const uint32_t fa = s_foff[t] + lead, fb = s_foff[t + 1] + lead;
        uint32_t b = t == 0 ? 0u : (fa + 15u) >> 4;
        for (; 16u * b < fb && b < nblk; b++)
            s_owner[b] = (uint8_t)t;
    }
    mbar_wait(&s_bar, 0);
    __syncthreads();
    const uint32_t *sw = reinterpret_cast<const uint32_t *>(smem);
    /* Phase 1: blocks inside one path, path-again or payload segment; Phase 2: the listed rest, segment by segment */
    uint16_t *s_list = reinterpret_cast<uint16_t *>(s_owner + ((nblk + 15u) & ~15u));
    if (t == 0)
        s_nlist = 0;
    __syncthreads();
    for (uint32_t b = t; b < nblk; b += JUTE_THREADS) {
        const int32_t bstart = (int32_t)(16u * b) - (int32_t)lead;
        const uint4 rc = s_rec[s_owner[b]];
        const uint32_t fo_b = (uint32_t)bstart - rc.x;
        const uint32_t Pi = rc.w & 0xFFFFu, Ji = rc.w >> 16;
        const uint32_t e0 = rc.y >> 24, e1 = e0 + Pi, e2 = e1 + F1, e3 = e2 + (PAIR ? Pi : 0u), e4 = e3 + F2, e5 = e4 + Ji;
        const bool whole = bstart >= 0 && (uint32_t)bstart + 16u <= total;
        const bool in_path = fo_b >= e0 && fo_b + 16u <= e1;
        const bool in_path2 = PAIR && fo_b >= e2 && fo_b + 16u <= e3;
        const bool in_data = DATA && fo_b >= e4 && fo_b + 16u <= e5;
        if (whole && (in_path || in_path2 || in_data)) {
            const uint32_t ys = rc.y & 0xFFFFFFu, zs = rc.z & 0xFFFFFFu;
            const uint32_t src = in_path ? ys + (fo_b - e0) : in_path2 ? ys + (fo_b - e2) : zs + (fo_b - e4);
            uint32_t v[4];
            load16(sw, src, v);
            stg_v4(p.out_bytes + a0 + 16ull * b, make_uint4(v[0], v[1], v[2], v[3]));
        } else {
            s_list[atomicAdd(&s_nlist, 1u)] = (uint16_t)b;
        }
    }
    __syncthreads();
    const uint32_t nlist = s_nlist;
    for (uint32_t li = t; li < nlist; li += JUTE_THREADS) {
        const uint32_t b = s_list[li];
        const int32_t bstart = (int32_t)(16u * b) - (int32_t)lead;
        uint32_t pos = bstart < 0 ? 0u : (uint32_t)bstart;
        const uint32_t end = min((uint32_t)(bstart + 16), total);
        uint32_t i = s_owner[b];
        uint32_t acc[4] = {0u, 0u, 0u, 0u};
        while (pos < end) {
            const uint4 rc = s_rec[i];
            const uint32_t fo_b = pos - rc.x;
            const uint32_t Pi = rc.w & 0xFFFFu, Ji = rc.w >> 16;
            const uint32_t e0 = rc.y >> 24, e1 = e0 + Pi, e2 = e1 + F1, e3 = e2 + (PAIR ? Pi : 0u), e4 = e3 + F2, e5 = e4 + Ji;
            const uint32_t e6 = e5 + (rc.z >> 24);
            const uint32_t ys = rc.y & 0xFFFFFFu, zs = rc.z & 0xFFFFFFu;
            const uint32_t fs = HDR + JUTE_ESLOT * i + 32u - e0;        /* framing byte k of the entry */
            uint32_t src, seg_end;
            if (fo_b < e0) {
                src = fs + fo_b;
                seg_end = e0;
            } else if (fo_b < e1) {
                src = ys + (fo_b - e0);
                seg_end = e1;
            } else if (PAIR && fo_b < e2) {
                src = fs + (fo_b - Pi);
                seg_end = e2;
            } else if (PAIR && fo_b < e3) {
                src = ys + (fo_b - e2);
                seg_end = e3;
            } else if (DATA && fo_b < e4) {
                src = fs + (fo_b - PM * Pi);
                seg_end = e4;
            } else if (DATA && fo_b < e5) {
                src = zs + (fo_b - e4);
                seg_end = e5;
            } else {
                src = fs + (fo_b - PM * Pi - Ji);
                seg_end = e6;
            }
            const uint32_t n = min(seg_end - fo_b, end - pos);
            const uint32_t d = (uint32_t)((int32_t)pos - bstart);
            uint32_t v[4];
            load16(sw, src - d, v);
            const uint4 mg = s_ge[d], ml = s_lt[d + n];
            acc[0] |= v[0] & mg.x & ml.x;
            acc[1] |= v[1] & mg.y & ml.y;
            acc[2] |= v[2] & mg.z & ml.z;
            acc[3] |= v[3] & mg.w & ml.w;
            pos += n;
            if (fo_b + n == e6)
                i++;
        }
        uint8_t *gp = p.out_bytes + a0 + 16ull * b;
        if (bstart >= 0 && (uint32_t)bstart + 16u <= total) {
            stg_v4(gp, make_uint4(acc[0], acc[1], acc[2], acc[3]));
        } else {
            const uint32_t d0 = bstart < 0 ? (uint32_t)(-bstart) : 0u, d1 = end - (uint32_t)max(bstart, 0) + d0;
            for (uint32_t k = d0; k < d1; k++)
                gp[k] = (uint8_t)(acc[k >> 2] >> (8u * (k & 3u)));
        }
    }
}

}  /* namespace regk */
#endif /* REGK_JUTE_CUH */
