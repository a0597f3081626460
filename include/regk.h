/*
 * regk.h — C-ABI of libregk.so, the H100-native replacement for registrar's
 * per-record registration hot path (SURVEY.md §8 rows A1–A5).
 *
 * The reference has no FFI of its own (it is 100 % JavaScript); the entry
 * points below are what an N-API addon for that path binds (see
 * INTEGRATION.md and registrar_b200/napi/).  Each one names the reference
 * code it replaces, relative to /root/reference:
 *
 *   regk_register_batch  <- lib/register.js:34-39   domainToPath()            (A1)
 *                           lib/register.js:221-223 path.join(p, hostname)    (A2)
 *                           lib/register.js:141-155 host-record object        (A3)
 *                           lib/register.js:156-159 zk.create(n,_obj,...) ->
 *                             zkplus JSON.stringify(_obj) -> UTF-8 bytes      (A4)
 *                           (new) per-record output offsets                   (A5)
 *   regk_set_types       <- lib/register.js:142,152 `type` / `_obj[type]` key
 *   REGK_NODE_ALIAS      <- lib/register.js:223     aliases.map(domainToPath)
 *
 * Conventions: extern "C", plain pointers and sizes, no exceptions cross the
 * boundary, every call returns a REGK_* status and leaves a message readable
 * through regk_last_error().  There is NO CPU fallback: without a usable
 * CUDA device regk_create() fails.
 *
 * Threading: a context is single-owner (one host thread at a time, one CUDA
 * stream).  The N-API shim runs calls on a napi_async_work thread and
 * resolves the Node errback on the main loop.
 */
#ifndef REGK_H
#define REGK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define REGK_ABI_VERSION 3

/* ---- status codes ------------------------------------------------------ */
#define REGK_OK                 0
#define REGK_ERR_INVALID_ARG    1   /* NULL pointer, bad flag combination, misaligned device pointer */
#define REGK_ERR_CUDA           2   /* CUDA runtime error; text in regk_last_error() */
#define REGK_ERR_OUT_OF_DOMAIN  3   /* >=1 record outside the fenced input domain; nothing is returned (unless the
                                       batch has REGK_SKIP_BAD: then only REGK_BAD_TOO_LARGE refuses it) */
#define REGK_ERR_NOMEM          4
#define REGK_ERR_STATE          5   /* e.g. type table not set, result already released */

/* ---- batch flags -------------------------------------------------------- */
#define REGK_IN_DEVICE   (1u << 0)  /* batch arrays are device pointers (16-byte aligned); else host memory */
#define REGK_OUT_DEVICE  (1u << 1)  /* result arrays are device pointers; else library-owned pinned host memory */
#define REGK_NODE_ALIAS  (1u << 2)  /* alias nodes: path = domainToPath(domain) un-normalised, no hostname
                                       (lib/register.js:223); default = host nodes (A2, lib/register.js:222) */
#define REGK_NO_JSON     (1u << 3)  /* paths only (skip A3/A4) */
#define REGK_NO_PATH     (1u << 4)  /* payloads only (skip A1/A2) */
#define REGK_JOB_STEP    (1u << 5)  /* this batch is the calling rank's shard of the multi-GPU job bound with
                                       regk_job_bind(): results go straight into every rank's whole-job buffers
                                       (requires REGK_IN_DEVICE | REGK_OUT_DEVICE, paths and payloads) */
#define REGK_SKIP_BAD    (1u << 6)  /* skip mode: a record whose only faults are value-fence bits (REGK_BAD_DOMAIN_BYTE,
                                       _HOST_BYTE, _ADDR_BYTE, _TYPE_ID) gets an empty path and payload (off[i] ==
                                       off[i+1]), every other record is composed exactly as in a batch of the kept records
                                       alone, and the call returns REGK_OK; bad_bits / first_bad then describe the skipped
                                       records and regk_skipped_records() lists them.  REGK_BAD_TOO_LARGE still refuses
                                       the whole batch.  Not with REGK_JOB_STEP.  A clean batch runs exactly the kernels
                                       of a plain one; a dirty one is composed a second time (DESIGN.md section 4) */

/* ---- per-record validation bits (regk_result.bad_bits) ------------------ */
#define REGK_BAD_DOMAIN_BYTE  (1u << 0)  /* byte >= 0x80 or '/' in a domain (JS toLowerCase / path.normalize
                                            semantics are only restated for ASCII, slash-free labels) */
#define REGK_BAD_HOST_BYTE    (1u << 1)  /* hostname empty, ".", "..", or has byte >= 0x80, NUL or '/' */
#define REGK_BAD_ADDR_BYTE    (1u << 2)  /* address empty (a falsy adminIp means auto-detect, register.js:143), or a byte
                                            outside 0x20..0x7f or needing a JSON escape (" or \) */
#define REGK_BAD_TYPE_ID      (1u << 3)  /* type_id >= number of types set */
#define REGK_BAD_TOO_LARGE    (1u << 4)  /* a single record's path or payload exceeds 2^31 bytes */
#define REGK_BAD_SERVICE_BYTE (1u << 5)  /* service records: srvce / proto byte outside 0x20..0x7f or needing a JSON escape */
#define REGK_BAD_KEY_ORDER    (1u << 6)  /* service records: key_order is not a permutation of the four members */

#define REGK_TTL_ABSENT  INT32_MIN      /* registration.ttl === undefined -> key omitted (register.js:144) */

typedef struct regk_ctx regk_ctx;

/*
 * One batch of service records, struct-of-arrays.  All offset arrays are CSR
 * style with n+1 entries, offsets in bytes (or elements for ports_off)
 * relative to the matching *_bytes / ports base.
 */
typedef struct regk_batch {
    uint64_t        n;              /* number of records */
    uint32_t        flags;          /* REGK_IN_DEVICE | REGK_OUT_DEVICE | REGK_NODE_ALIAS | ... */
    uint32_t        host_stride;    /* used when host_off == NULL: hostname i = host_bytes[i*stride, +stride) */

    /* Lengths of the packed arrays (== the last entry of the matching offset array).  Required for
       device-resident batches (the library does not read device memory to size its outputs);
       may be 0 for host batches, the library then reads them from the offset arrays. */
    uint64_t        domain_bytes_len;
    uint64_t        host_bytes_len;
    uint64_t        addr_bytes_len;
    uint64_t        ports_len;      /* elements */

    const uint8_t  *domain_bytes;   /* opts.domain (or one alias) per record, packed */
    const uint32_t *domain_off;     /* [n+1] */

    const uint8_t  *host_bytes;     /* os.hostname() per record (zone UUID in Triton); ignored for alias nodes */
    const uint32_t *host_off;       /* [n+1] or NULL for fixed stride */

    const uint8_t  *type_id;        /* [n] index into the table given to regk_set_types() */

    const uint8_t  *addr_bytes;     /* opts.adminIp per record, packed */
    const uint32_t *addr_off;       /* [n+1] */

    const int32_t  *ttl;            /* [n]; REGK_TTL_ABSENT = undefined */

    const uint32_t *ports_off;      /* [n+1] element offsets into ports, or NULL = no record has ports */
    const uint32_t *ports;          /* registration.ports (or [service.service.port]) values */
    const uint8_t  *ports_present;  /* [n] or NULL.  NULL: ports key present iff k>0.  Non-NULL: !=0 means
                                       present, so an empty array is emitted as "ports":[] (register.js:146) */
} regk_batch;

/*
 * Result views.  path_bytes[path_off[i] .. path_off[i+1]) is znode path i,
 * json_bytes[json_off[i] .. json_off[i+1]) is payload i (what zkplus would
 * hand to ZooKeeper).  Owned by the context until regk_release() or the next
 * regk_register_batch() on the same context with the same result slot.
 */
typedef struct regk_result {
    uint64_t        n;
    uint32_t        flags;          /* REGK_OUT_DEVICE if the pointers below are device pointers */
    uint32_t        bad_bits;       /* OR of REGK_BAD_* over all records (0 on success) */
    uint64_t        first_bad;      /* smallest offending record index when bad_bits != 0 */
    uint8_t        *path_bytes;
    uint64_t       *path_off;       /* [n+1] */
    uint64_t        path_total;     /* == path_off[n] */
    uint8_t        *json_bytes;
    uint64_t       *json_off;       /* [n+1] */
    uint64_t        json_total;     /* == json_off[n] */
    float           kernel_ms;      /* device time of all kernels of the batch (CUDA events on the ctx stream) */
    float           path_kernel_ms; /* regk_path_kernel */
    float           json_kernel_ms; /* regk_json_kernel */
    float           json_len_kernel_ms; /* regk_json_len_kernel (payload lengths + tile bases) */
    uint32_t        launches;       /* kernels launched by this call */
    void           *opaque;         /* library bookkeeping */
    /* REGK_JOB_STEP only: where this rank's shard sits in the job-wide streams and how long those are.  The
       result pointers above are then the rank's own WHOLE-JOB buffers (offsets job-absolute, n_total + 1
       entries); path_total / json_total stay the shard's own byte counts. */
    uint64_t        job_path_base, job_path_total;
    uint64_t        job_json_base, job_json_total;
    uint32_t        generic_tiles;  /* tiles (128 records, counted per kernel) that did not fit the kernels' shared-memory
                                       budget and were composed straight from / to global memory (about 10x slower) */
    uint32_t        reserved;
    /* option "offsets32" = 1 (host results only, both streams below 4 GiB): the offsets come back as 32-bit arrays
       - half the device-to-host bytes of the two offset arrays - and path_off / json_off are NULL */
    uint32_t       *path_off32;     /* [n+1] */
    uint32_t       *json_off32;     /* [n+1] */
} regk_result;

/* ---- lifecycle ----------------------------------------------------------- */
int         regk_abi_version(void);
int         regk_create(int device, regk_ctx **out);   /* binds one CUDA device; fails if none */
void        regk_destroy(regk_ctx *ctx);
const char *regk_last_error(const regk_ctx *ctx);      /* ctx may be NULL: error of the last failed regk_create */

/* Run on a caller-supplied cudaStream_t (e.g. torch's current stream); NULL = the context's own non-blocking
 * stream.  The legacy default stream must be named explicitly (cudaStreamLegacy, (void *)0x1): a NULL here does
 * NOT mean "stream 0", and work on the own stream is not ordered with work on the default stream. */
int         regk_set_stream(regk_ctx *ctx, void *cuda_stream);

/*
 * Record-type table (registration.type values).  Strings are arbitrary UTF-8;
 * JSON escaping (ECMA-262 QuoteJSONString) is applied here, on the host, once.
 * Rejected (REGK_ERR_OUT_OF_DOMAIN): "type", "address", "ttl" (the dynamic key
 * would overwrite a fixed one, register.js:152), "__proto__", canonical
 * array-index strings ("0", "42": V8 orders integer keys first), and bytes
 * that are not well-formed UTF-8 (overlong forms, encoded surrogates, code
 * points above U+10FFFF, truncated sequences, stray continuation bytes): no JS
 * string has such a UTF-8 form, so the reference could never write them.
 * Rejected (REGK_ERR_INVALID_ARG): more than 255 types, or a fragment table
 * over 16 KB (each type takes eight copies of its escaped name plus about 200
 * bytes: one name of up to about 2000 escaped bytes, or about 80 short names).
 * A rejected call leaves the previous table in force.
 */
int         regk_set_types(regk_ctx *ctx, const char *const *types, const uint32_t *lens, uint32_t ntypes);

/* ---- the hot path ------------------------------------------------------ */
int         regk_register_batch(regk_ctx *ctx, const regk_batch *batch, regk_result *result);
/* With option "async" = 1 regk_register_batch() only enqueues; regk_finish() waits for that batch,
   fills totals / validation / timings and returns its status.  (Synchronous mode calls it itself.) */
int         regk_finish(regk_ctx *ctx, regk_result *result);
int         regk_release(regk_ctx *ctx, regk_result *result);

/*
 * ---- service records (reference lib/register.js:45-75 registerService) ------------------------------------------
 * The persistent node a registration with `registration.service` also writes: zk.put(domainToPath(domain),
 * { type: 'service', service: registration.service }) with registration.service = { type: 'service', service:
 * { srvce, proto, port, ttl } } (asserted at :186-199, ttl defaulted to 60 at :197).  Payload bytes (zkplus ->
 * JSON.stringify, insertion order):
 *   {"type":"service","service":{"type":"service","service":{<srvce, proto, port, ttl in the CALLER's key order>}}}
 * The node's PATH is an alias-mode path (regk_register_batch with REGK_NODE_ALIAS | REGK_NO_JSON).
 * key_order[i]: four 2-bit key ids, first member in bits 0-1 (0 srvce, 1 proto, 2 port, 3 ttl); NULL = that order.
 * A ttl the caller left undefined is appended last by the reference's assignment: the host layer passes the
 * defaulted value and an order that ends in ttl.  Fence: REGK_BAD_SERVICE_BYTE, REGK_BAD_KEY_ORDER,
 * REGK_BAD_TOO_LARGE (offsets); port is uint32, ttl int32.  Only json_bytes / json_off / json_total of the result
 * are filled.  Synchronous; honours REGK_IN_DEVICE / REGK_OUT_DEVICE.
 */
typedef struct regk_service_batch {
    uint64_t        n;
    uint32_t        flags;
    uint32_t        reserved;
    uint64_t        srvce_bytes_len, proto_bytes_len;   /* required for device batches */
    const uint8_t  *srvce_bytes;    /* registration.service.service.srvce per record, packed ("_http") */
    const uint32_t *srvce_off;      /* [n+1] */
    const uint8_t  *proto_bytes;    /* ....proto ("_tcp") */
    const uint32_t *proto_off;      /* [n+1] */
    const uint32_t *port;           /* [n] */
    const int32_t  *ttl;            /* [n] (already defaulted) */
    const uint8_t  *key_order;      /* [n] or NULL */
} regk_service_batch;

int         regk_service_records(regk_ctx *ctx, const regk_service_batch *batch, regk_result *result);

/*
 * ---- the records a REGK_SKIP_BAD batch skipped ----------------------------------------------------------------
 * Describes the batch finished last on this context, which must have been a skip-mode batch (else REGK_ERR_STATE).
 * The list is compact: a few bad records in 10^7 cost a few bytes, not an n-byte mask.  Downstream calls on "the
 * batch finished last" (regk_parent_dirs, regk_jute_frames / regk_jute_requests, regk_decode with REGK_DECODE_LAST)
 * see the KEPT records in order: their record k is the k-th kept record.  flags: REGK_OUT_DEVICE returns device
 * pointers, otherwise pinned host arrays; both stay valid until the next batch on the context.
 */
typedef struct regk_skipped {
    uint64_t n;                     /* records of the batch */
    uint64_t n_skipped;
    uint32_t flags;                 /* REGK_OUT_DEVICE: device pointers, else pinned host arrays */
    uint32_t bad_bits;              /* OR over the skipped records */
    const uint64_t *index;          /* [n_skipped] ascending record indices */
    const uint8_t  *bits;           /* [n_skipped] REGK_BAD_* of each */
} regk_skipped;

int         regk_skipped_records(regk_ctx *ctx, uint32_t flags, regk_skipped *out);

/* Pinned host memory for callers that want zero-staging H2D/D2H. */
void       *regk_host_alloc(regk_ctx *ctx, size_t bytes);
void        regk_host_free(regk_ctx *ctx, void *p);

/* Device memory helpers for non-CUDA hosts (Node, ctypes). */
void       *regk_dev_alloc(regk_ctx *ctx, size_t bytes);
void        regk_dev_free(regk_ctx *ctx, void *p);
int         regk_memcpy_h2d(regk_ctx *ctx, void *dst_dev, const void *src_host, size_t bytes);
int         regk_memcpy_d2h(regk_ctx *ctx, void *dst_host, const void *src_dev, size_t bytes);
int         regk_sync(regk_ctx *ctx);

/*
 * ---- multi-GPU reassembly (BASELINE.json configs[3]: "sharded across 8 GPUs, all-gather of the output byte
 * stream") ---------------------------------------------------------------------------------------------------
 * One process per GPU; every rank owns whole-job result buffers (regk_dev_alloc) that its peers map through
 * CUDA IPC.  regk_gather_push is an all-gather-v written as ONE kernel over NVLink/NVSwitch peer memory: the
 * calling rank stores its shard's path / payload bytes at their final positions in EVERY rank's buffers
 * (16-byte stores, re-aligned to each destination) and its record offsets rebased by the bytes of the ranks
 * before it.  The reference has no counterpart (one registrar process per host); the operation it replaces is
 * "concatenate the shards' results in record order" (SURVEY.md §8e).
 */
#define REGK_IPC_HANDLE_BYTES 64
#define REGK_MAX_PEERS 16

/* Export a device allocation made by regk_dev_alloc / map a peer's export into this process / unmap it. */
int         regk_ipc_export(regk_ctx *ctx, const void *dev_ptr, unsigned char handle[REGK_IPC_HANDLE_BYTES]);
int         regk_ipc_open(regk_ctx *ctx, const unsigned char handle[REGK_IPC_HANDLE_BYTES], void **peer_ptr);
int         regk_ipc_close(regk_ctx *ctx, void *peer_ptr);

typedef struct regk_gather {
    uint32_t world, rank;
    uint64_t rec_base;              /* records held by the ranks before this one */
    uint64_t n_total;               /* records of the whole job */
    const uint64_t *totals;         /* DEVICE [world][2]: {path bytes, payload bytes} of every rank's shard, as
                                       all-gathered by the caller on the context's stream */
    void *path_bytes[REGK_MAX_PEERS];       /* rank q's whole-job buffers as mapped in THIS process ([rank] = own) */
    uint64_t *path_off[REGK_MAX_PEERS];     /* uint64 [n_total + 1] */
    void *json_bytes[REGK_MAX_PEERS];
    uint64_t *json_off[REGK_MAX_PEERS];
    uint64_t path_cap, json_cap;    /* bytes behind every whole-job byte buffer */
} regk_gather;

/* Enqueue the push of `shard` (a finished REGK_OUT_DEVICE result of this context) on the context's stream.
 * Remote data is complete on a rank once every rank's push has finished: follow it with a stream-ordered
 * barrier across ranks (e.g. a 1-element NCCL all-reduce).  Out-of-range totals raise REGK_ERR_INVALID_ARG
 * at regk_sync time through the returned device flag, never a wild store. */
int         regk_gather_push(regk_ctx *ctx, const regk_result *shard, const regk_gather *g);

/*
 * ---- the multi-GPU job with the all-gather FUSED into the compose kernels ---------------------------------------
 * BASELINE.json configs[3]/[4]: "the record batch shards across the GPUs of one box, one all-gather reassembles
 * the output byte stream".  Here the reassembly is not a separate pass: every rank's regk_path_kernel /
 * regk_json_kernel place each tile at its FINAL position of the job-wide stream and store it, straight out of
 * shared memory (TMA bulk copies, byte-masked at the tile's ragged ends), into the whole-job buffers of ALL ranks
 * over NVLink / NVSwitch, offsets included.  What the ranks must know of each other is two numbers per shard - its
 * path bytes (closed form in the input sizes) and its payload bytes (known after the path kernel's side job) - and
 * those travel through a peer-memory mailbox (regk_peersync.cuh): a 16-byte all-gather + barrier written as a
 * one-warp kernel, no library collective on the data path.  One step on every rank:
 *     exchange(path totals)  ->  regk_path_kernel (push)  ->  exchange(payload totals)  ->  regk_json_kernel (push)
 *     ->  exchange (closing barrier: every rank's stores have landed everywhere)
 * all enqueued on the context's stream by ONE regk_register_batch(REGK_JOB_STEP) call.  The first exchange doubles
 * as the entry barrier: a rank starts overwriting its peers' buffers only after every rank's stream has reached
 * this step, i.e. has finished whatever it had enqueued on the previous step's results.
 * A shard with empty labels (path.join drops them, so the closed-form placement fails) is refused with
 * REGK_ERR_STATE at regk_finish: run it unfused (plain batch + regk_gather_push).
 */
#define REGK_MAILBOX_BYTES (REGK_MAX_PEERS * 32)    /* one 32-byte slot per sender; zero it once after allocation */

typedef struct regk_job {
    uint32_t world, rank;
    uint64_t rec_base;              /* records held by the ranks before this one */
    uint64_t n_total;               /* records of the whole job */
    void *path_bytes[REGK_MAX_PEERS];       /* rank q's whole-job buffers as mapped in THIS process ([rank] = own) */
    uint64_t *path_off[REGK_MAX_PEERS];     /* uint64 [n_total + 1] */
    void *json_bytes[REGK_MAX_PEERS];
    uint64_t *json_off[REGK_MAX_PEERS];
    uint64_t *mailbox[REGK_MAX_PEERS];      /* REGK_MAILBOX_BYTES each, zeroed once */
    uint64_t path_cap, json_cap;    /* bytes behind every whole-job byte buffer */
    uint64_t timeout_ms;            /* how long an exchange waits for a silent peer before failing (0 = 10 s) */
} regk_job;

/* Bind (copy) the job description to the context; NULL unbinds.  No batch may be pending. */
int         regk_job_bind(regk_ctx *ctx, const regk_job *job);

/*
 * ---- setupDirectories for a batch (reference lib/register.js:107-125: mkdirp(path.dirname(n)) for every node) ----
 * Works on the path stream of the batch most recently finished on this context (its device copy is still in
 * the context).  parent_len[i] = byte length of path.dirname(path_i), always a prefix of path_i (node >= 6
 * posix semantics: '/' for a top-level node, '//' when the last separator sits at index 1); unique_first[] =
 * record index of the first occurrence of every DISTINCT directory, ascending - the set a batched mkdirp
 * needs (10^7 instances share ~10^3 parents).  Directories are compared byte for byte; hashing only picks a
 * table slot.  flags: REGK_OUT_DEVICE returns device pointers, otherwise pinned host arrays; both stay valid
 * until the next regk_parent_dirs call on the context.
 */
typedef struct regk_parents {
    uint64_t n;                     /* records of the batch */
    uint64_t n_unique;
    uint32_t flags;
    uint32_t launches;
    const uint32_t *parent_len;     /* [n] */
    const uint64_t *unique_first;   /* [n_unique] */
    float kernel_ms;
} regk_parents;

int         regk_parent_dirs(regk_ctx *ctx, uint32_t flags, regk_parents *out);

/*
 * ---- ZooKeeper wire framing of a batch (reference lib/register.js:156-159: zk.create(n, _obj, {flags:
 * ['ephemeral_plus']}) -> zkplus -> one jute CreateRequest per node on the socket) -----------------------------------
 * Works on the batch most recently finished on this context (paths AND payloads; its device copies are still in
 * the context): frame i = 4-byte big-endian length | RequestHeader{xid = xid_base + i, type = 1 (create)} |
 * CreateRequest{path, data = payload i, acl = [OPEN_ACL_UNSAFE: perms 31, "world", "anyone"], flags = zk_flags}
 * (1 = EPHEMERAL for host records, 0 = persistent for service records).  frame_off[i] = path_off[i] + json_off[i]
 * + 51 i.  PARITY UNPINNED: zkplus / ZooKeeper are not in the reference tree (package.json:20); the layout follows
 * the published zookeeper.jute definitions and is tested against an independent restatement, not against a server.
 * flags: REGK_OUT_DEVICE returns device pointers, else pinned host arrays; valid until the next call.
 */
typedef struct regk_frames {
    uint64_t n;
    uint64_t total;                 /* == frame_off[n] */
    uint32_t flags;
    uint32_t launches;
    const uint8_t *frame_bytes;
    const uint64_t *frame_off;      /* [n+1] */
    float kernel_ms;
} regk_frames;

int         regk_jute_frames(regk_ctx *ctx, uint32_t flags, int32_t xid_base, uint32_t zk_flags, regk_frames *out);

/*
 * The other requests of register()'s choreography, and transactions.  Same batch, same kernel, other framing:
 *   REGK_ZK_CREATE   as regk_jute_frames (lib/register.js:156-159 create; :62 put on a node that does not exist yet)
 *   REGK_ZK_DELETE   DeleteRequest{path, version}: the unlink list of cleanupPreviousEntries (lib/register.js:85-95)
 *                    - one request per node path of the batch, no payload stream needed
 *   REGK_ZK_SETDATA  SetDataRequest{path, data, version}: zkplus put() on an existing node (lib/register.js:62)
 * group = 0: one request per record, xid = xid_base + i.  group = g >= 1: ZooKeeper multi transactions (OpCode 14) of g
 * operations each (the last one may be shorter): frame k = len | xid_base + k | 14 | g x { MultiHeader{op, done = false,
 * err = -1} | request body } | MultiHeader{-1, true, -1} - registering a whole fleet atomically in n / g round trips.
 * out->n = number of frames, frame_off has n + 1 entries.  version is -1 ("any") unless the caller tracks versions.
 * PARITY UNPINNED like regk_jute_frames: restated from zookeeper.jute / MultiTransactionRecord, tested against an
 * independent restatement (oracle/pyoracle.py), not against a server.
 *   REGK_ZK_GETDATA  GetDataRequest{path, watch = false}: the heartbeat's read of every node (lib/zk.js:21-44), whose
 *                    replies regk_read_replies turns into a snapshot.  Frame i = len | xid_base + i (wrapping) | 4 | path
 *                    length | path | 0, 17 + P_i bytes.  Paths only; group != 0 is REGK_ERR_INVALID_ARG (a multi holds
 *                    no reads).  A successful call records the batch, xid_base and n for regk_read_replies.
 *   REGK_ZK_EXISTS   ExistsRequest{path, watch = false}: the reference's own heartbeat request, zk.stat per node
 *                    (lib/zk.js:30-35), whose replies regk_read_stats reads.  The getData layout with op word 3: frame i =
 *                    len | xid_base + i (wrapping) | 3 | path length | path | 0, 17 + P_i bytes; group != 0 is
 *                    REGK_ERR_INVALID_ARG.  The frames carry paths only, but the batch must have its payload stream too
 *                    (REGK_ERR_STATE otherwise): regk_reconcile_stats classes the replies against the payload lengths.
 *                    A successful call records the batch, xid_base and n in fields of its own, so an exists framing
 *                    and a getData framing of one batch can both be outstanding (the frames share one buffer: copy or
 *                    send the first before framing the second).  Like getData it leaves regk_read_results' record of
 *                    the last write framing in force.
 */
#define REGK_ZK_CREATE  1u
#define REGK_ZK_DELETE  2u
#define REGK_ZK_EXISTS  3u
#define REGK_ZK_GETDATA 4u
#define REGK_ZK_SETDATA 5u

typedef struct regk_jute_opts {
    uint32_t op;                    /* REGK_ZK_* */
    uint32_t flags;                 /* REGK_OUT_DEVICE */
    int32_t xid_base;
    uint32_t zk_flags;              /* create: CreateMode bits (1 = EPHEMERAL) */
    int32_t version;                /* delete / setData: expected version, -1 = any */
    uint32_t group;                 /* 0: single requests; g >= 1: multi transactions of g operations */
} regk_jute_opts;

int         regk_jute_requests(regk_ctx *ctx, const regk_jute_opts *opts, regk_frames *out);

/*
 * ---- the whole mkdirp set of a batch (reference lib/register.js:107-129: zk.mkdirp(path.dirname(n)) for every node;
 * mkdirp creates the directory AND every ancestor, and ZooKeeper creates no node whose parent is missing) -----------
 * Works on the path stream of the batch finished last, as regk_parent_dirs does: a skip-mode batch contributes its
 * kept records in order; a REGK_NO_PATH batch, an empty batch (it leaves no path stream), a REGK_JOB_STEP result or a
 * pending batch is REGK_ERR_STATE.
 * D_i = path.dirname(path_i) (parent_len of regk_parent_dirs).  D_i == "/" creates nothing.  D_i is INVALID when
 * ZooKeeper's path check rejects it - an empty component ("//"), a trailing '/', or a byte in 0x00-0x1F or 0x7F
 * (only alias nodes with empty labels and domains with control bytes get there): it contributes nothing and its
 * first record is listed in invalid[].  Every other D_i contributes each of its prefixes that ends at a component
 * boundary: /a, /a/b, ..., D_i.  The set is the union, each directory once, in a deterministic order: ascending
 * depth (components), then ascending first record whose directory has it as a prefix - every parent precedes its
 * children, so the whole list can be pipelined on one session.  Directory k = path_{dir_rec[k]}[0, dir_len[k]), also
 * packed as dir_bytes[dir_off[k], dir_off[k+1]).  Bytes are compared byte for byte; a hash only picks a table slot.
 * flags: REGK_OUT_DEVICE returns device pointers, else pinned host arrays; they stay valid until the next
 * regk_mkdirp_dirs call (a later batch does not touch them).  Option "mkdirp_tight_table" = 1 shrinks the hash table
 * to the smallest power of two above the entry count (long probe chains; for testing).
 */
typedef struct regk_dirs {
    uint64_t n;                     /* records of the batch */
    uint64_t n_dirs;                /* directories to create */
    uint64_t n_invalid;             /* distinct immediate directories ZooKeeper would reject */
    uint32_t flags;                 /* REGK_OUT_DEVICE */
    uint32_t launches;
    uint32_t max_depth;
    uint32_t reserved;
    const uint64_t *dir_rec;        /* [n_dirs] first record whose directory has this one as a prefix */
    const uint32_t *dir_len;        /* [n_dirs] */
    const uint64_t *depth_off;      /* [max_depth + 1] depth d is directories depth_off[d-1] .. depth_off[d]; [0] = 0 */
    const uint8_t  *dir_bytes;      /* [dir_bytes_len] packed directory paths */
    const uint64_t *dir_off;        /* [n_dirs + 1] */
    const uint64_t *invalid;        /* [n_invalid] first record of each rejected directory, ascending */
    uint64_t dir_bytes_len;
    float kernel_ms;                /* parent_ms + closure_ms + gather_ms */
    float parent_ms;                /* the distinct immediate directories (regk_parents.cuh kernels) */
    float closure_ms;               /* classify + every depth's passes, including the host's read of two counters per depth */
    float gather_ms;                /* dir_off and dir_bytes */
} regk_dirs;

int         regk_mkdirp_dirs(regk_ctx *ctx, uint32_t flags, regk_dirs *out);

/*
 * The mkdirp set of the last regk_mkdirp_dirs call (REGK_ERR_STATE without one) as ready-to-send frames: directory k
 * becomes len | RequestHeader{xid = xid_base + k (wrapping), type = 1} | CreateRequest{path, data = empty buffer
 * (length 0), acl = [OPEN_ACL_UNSAFE], flags = zk_flags}, in set order - the same kernel and layout as
 * regk_jute_requests(REGK_ZK_CREATE, group = 0).  Single requests only: a multi transaction would abort as a whole on
 * the first directory that already exists, and a NODE_EXISTS reply to one of these frames is expected (zkplus'
 * mkdirp tolerates it).  PARITY UNPINNED: the data bytes and flags zkplus' own mkdirp sends are not in the reference
 * tree (zkplus is a dependency, package.json:20), hence an empty buffer and zk_flags as a parameter (0 = persistent).
 * flags: REGK_OUT_DEVICE returns device pointers, else pinned host arrays; valid until the next call.  These buffers
 * are separate from regk_jute_requests', so the create frames of the batch and the mkdirp frames can be held together.
 */
int         regk_mkdirp_requests(regk_ctx *ctx, int32_t xid_base, uint32_t zk_flags, uint32_t flags, regk_frames *out);

/*
 * ---- the reader side: decode paths and payloads back into records (README.md:462-480, :587-664) -----------------
 * Inverse of regk_register_batch / regk_service_records for audits of registry contents and round-trip checks:
 *   path    -> domain (labels reversed back, '/' -> '.'); for host nodes the last component is the instance name
 *              (lib/register.js:221-223) and is reported as (host_pos, host_len) inside the path
 *   payload -> type, address (positions inside the payload), ttl, ports - for the canonical compact form
 *              {"type":T,"address":A[,"ttl":n],T:{"address":A[,"ports":[..]]}} ; service records
 *              {"type":"service","service":{"type":"service","service":{srvce,proto,port,ttl in any order}}} come
 *              back with type_* = srvce, addr_* = proto, ports[0] = port.
 * Input: explicit streams (host, or device with REGK_IN_DEVICE; 64-bit CSR offsets as in regk_result), or
 * REGK_DECODE_LAST = the batch finished last on this context.  Either stream may be NULL.
 * Output: rec[n]; domains in SLOT layout (domain i = dom_bytes[path_off[i], + rec[i].dom_len)); ports in slot layout
 * (record i's ports = ports[json_off[i] / 2, + rec[i].nports)).  REGK_OUT_DEVICE returns device pointers.
 */
#define REGK_DECODE_LAST       (1u << 8)

#define REGK_DEC_PATH_OK        (1u << 0)
#define REGK_DEC_HOST_RECORD    (1u << 1)
#define REGK_DEC_SERVICE_RECORD (1u << 2)
#define REGK_DEC_NOT_CANONICAL  (1u << 3)   /* not the compact form this library writes */
#define REGK_DEC_KEY_MISMATCH   (1u << 4)   /* the inner object's name differs from the value of "type" (README.md:596) */
#define REGK_DEC_ADDR_MISMATCH  (1u << 5)   /* the two "address" members differ */
#define REGK_DEC_BAD_NUMBER     (1u << 6)   /* ttl / port not an integer in range */
#define REGK_DEC_BAD_PATH       (1u << 7)   /* no leading '/', or a host node without an instance name */

typedef struct regk_decoded {
    uint32_t flags;                 /* REGK_DEC_* */
    uint32_t dom_len;
    uint32_t host_pos, host_len;    /* instance name inside the path (host nodes) */
    uint32_t type_pos, type_len;    /* inside the payload (JSON escapes left as they are) */
    uint32_t addr_pos, addr_len;
    int32_t  ttl;                   /* REGK_TTL_ABSENT when the key is missing */
    uint32_t nports;                /* 0xFFFFFFFF when the key is missing */
} regk_decoded;

typedef struct regk_decode_in {
    uint64_t n;
    uint32_t flags;                 /* REGK_IN_DEVICE | REGK_OUT_DEVICE | REGK_DECODE_LAST */
    uint32_t host_nodes;            /* != 0: paths are host nodes (domain path + '/' + instance name) */
    uint64_t path_total, json_total;    /* required for device streams */
    const uint8_t *path_bytes;
    const uint64_t *path_off;       /* [n+1] */
    const uint8_t *json_bytes;
    const uint64_t *json_off;       /* [n+1] */
} regk_decode_in;

typedef struct regk_decode_out {
    uint64_t n;
    uint32_t flags;
    uint32_t launches;
    const regk_decoded *rec;        /* [n] */
    const uint8_t *dom_bytes;       /* [path_total] slot layout */
    const uint32_t *ports;          /* [json_total / 2 + 1] slot layout */
    uint64_t dom_bytes_len, ports_len;
    float kernel_ms;
} regk_decode_out;

int         regk_decode(regk_ctx *ctx, const regk_decode_in *in, regk_decode_out *out);

/*
 * ---- reconcile a batch with a snapshot of the registry (the batch form of the reference's heartbeat check,
 * lib/zk.js:21-44 and lib/index.js:55-159: stat every node, register again what is missing) ----------------------
 * Desired = the batch finished last on this context, as for regk_jute_requests: paths AND payloads required; a
 * skip-mode batch contributes its kept records in order; no batch, a REGK_NO_PATH / REGK_NO_JSON batch, an empty batch
 * (it leaves no streams), a REGK_JOB_STEP result or a pending batch is REGK_ERR_STATE.
 * Observed = a snapshot of m nodes (path j, data j) in the layout regk_decode accepts: host streams, or device streams
 * with REGK_IN_DEVICE (bytes 4-byte aligned, offsets 8-byte aligned); u64 CSR offsets; path_total / json_total are
 * required for device streams; host_nodes is ignored, REGK_DECODE_LAST is REGK_ERR_INVALID_ARG.  Offsets that are not
 * monotone or reach past the totals are REGK_ERR_INVALID_ARG naming the smallest bad node (host snapshots are checked
 * on the host, device snapshots by the first kernel before any byte of that node is read).  A snapshot in which two
 * nodes have the same path is malformed (a registry cannot hold that): REGK_ERR_INVALID_ARG naming the later node.
 * The snapshot must cover exactly the namespace the batch owns: every node it holds that the batch does not produce -
 * directories included - is classed DELETE.
 * Nodes are keyed by their path bytes, compared byte for byte (a hash only picks a table slot); the class depends on
 * bytes alone (no ephemeral owners, no versions) - regk_reconcile_owned below also weighs each node's Stat.  Record i:
 *   REGK_DELTA_DUP     an earlier record of the batch has the same path (the first occurrence decides); no request
 *   REGK_DELTA_CREATE  no node has path i
 *   REGK_DELTA_UPDATE  the node with path i holds data that differs from payload i in length or in a byte
 *   REGK_DELTA_SAME    the node with path i holds payload i
 * match[i] = that node's index or UINT64_MAX (DUP records carry their path's match too).  Node j: REGK_DELTA_KEEP if
 * some record has path j, else REGK_DELTA_DELETE.  create / update / dup list record indices, del snapshot indices,
 * all ascending.  n and m must be < 2^32 - 1.  flags: REGK_OUT_DEVICE returns device pointers, else pinned host
 * arrays; valid until the next regk_reconcile call.
 * The call also gathers the three request sets (create paths + payloads, update paths + payloads, delete paths) into
 * streams of the library's own, so regk_reconcile_requests needs neither the snapshot nor the batch afterwards; a later
 * batch does not touch them.  Option "reconcile_tight_table" = 1 sizes both hash tables to the smallest power of two
 * above their entry count (long probe chains; for testing).
 */
#define REGK_DELTA_SAME   0u        /* cls[] */
#define REGK_DELTA_CREATE 1u
#define REGK_DELTA_UPDATE 2u
#define REGK_DELTA_DUP    3u
#define REGK_DELTA_KEEP   0u        /* obs_cls[] */
#define REGK_DELTA_DELETE 1u

typedef struct regk_delta {
    uint64_t n, m;                  /* records of the batch finished last / nodes of the snapshot */
    uint64_t n_same, n_create, n_update, n_dup, n_delete;
    uint32_t flags, launches;       /* REGK_OUT_DEVICE */
    const uint8_t  *cls;            /* [n] REGK_DELTA_SAME / _CREATE / _UPDATE / _DUP */
    const uint64_t *match;          /* [n] */
    const uint8_t  *obs_cls;        /* [m] REGK_DELTA_KEEP / _DELETE */
    const uint64_t *create, *update, *dup;   /* ascending record indices */
    const uint64_t *del;            /* [n_delete] ascending snapshot indices */
    float kernel_ms;
} regk_delta;

int         regk_reconcile(regk_ctx *ctx, const regk_decode_in *snapshot, uint32_t flags, regk_delta *out);

/*
 * The requests that repair the registry, from the last regk_reconcile call (REGK_ERR_STATE without one), framed
 * exactly as regk_jute_requests frames a batch: frame k is list entry k (group = 0) or multi transaction k, xid =
 * xid_base + k; group, version and zk_flags mean what they mean there.
 *   REGK_ZK_CREATE   the create list: CreateRequest{path i, payload i}
 *   REGK_ZK_SETDATA  the update list: SetDataRequest{path i, payload i, version}
 *   REGK_ZK_DELETE   the delete list: DeleteRequest{snapshot path j, version}
 * Send them in this order: delete, then the creates' parents (regk_mkdirp_dirs / regk_mkdirp_requests), then create,
 * then setData, then (after regk_reconcile_owned) replace.  flags: REGK_OUT_DEVICE returns device pointers, else pinned
 * host arrays; valid until the next call.  The frames come from whichever of regk_reconcile / regk_reconcile_owned last
 * succeeded.  After regk_reconcile_owned two more options exist:
 *   REGK_ZK_REPLACE           (op) the replace list: frame q is one multi transaction (group = 0 counts as 1; at most
 *                             32768 entries, i.e. 65536 operations) - len | xid_base + q | 14 | for each entry (record i):
 *                             MultiHeader{2, false, -1} DeleteRequest{path i, version} MultiHeader{1, false, -1}
 *                             CreateRequest{path i, payload i, [OPEN_ACL_UNSAFE], zk_flags} | MultiHeader{-1, true, -1}.
 *                             Entry r is 65 + 2 P + J bytes, a frame 21 more.  The node is never missing: ZooKeeper applies
 *                             the delete and the create together or neither.
 *   REGK_ZK_VERSION_OBSERVED  (flags) every delete, setData and the delete of a replace carries the Stat.version its
 *                             node had in the snapshot instead of opts->version: the write fails with BADVERSION if the
 *                             node changed since.  Not with REGK_ZK_CREATE (REGK_ERR_INVALID_ARG).
 * Both are REGK_ERR_STATE after a plain regk_reconcile.  After regk_reconcile_owned, REGK_ZK_CREATE and REGK_ZK_REPLACE
 * require opts->zk_flags == the zk_flags the reconcile classified with (REGK_ERR_INVALID_ARG otherwise): a node created
 * in another mode would be classed REPLACE again by the next reconcile, and the repair would never converge.
 */
#define REGK_ZK_REPLACE          256u       /* regk_jute_opts.op: not a ZooKeeper OpCode */
#define REGK_ZK_VERSION_OBSERVED (1u << 9)  /* regk_jute_opts.flags */
/* regk_jute_opts.flags: the read framings (regk_jute_requests with REGK_ZK_EXISTS / REGK_ZK_GETDATA,
   regk_children_requests with REGK_ZK_GETCHILDREN) write the request's trailing watch byte as 1 instead of 0, so the
   server arms a one-shot watch on each node or directory and later pushes a WatcherEvent when it changes (read by
   regk_read_events).  Without the flag every frame is byte for byte what it was.  With any write op (create, delete,
   setData, replace; regk_reconcile_requests; regk_children_requests' delete) it is REGK_ERR_INVALID_ARG. */
#define REGK_ZK_WATCH            (1u << 10)

int         regk_reconcile_requests(regk_ctx *ctx, const regk_jute_opts *opts, regk_frames *out);

/*
 * ---- reconcile against node stats: ephemeral owners and versions (the reference re-registers after a session loss by
 * unlinking every node, waiting 1 s and creating it again, lib/register.js:85-95, :228-239) ----------------------------
 * As regk_reconcile, with the Stat of every snapshot node, as the caller's client read it (getData / exists replies):
 * version[j] = Stat.version, ephemeral_owner[j] = Stat.ephemeralOwner (0 = persistent).  The arrays live where the
 * snapshot's streams do (device arrays with REGK_IN_DEVICE: version 4-byte, ephemeral_owner 8-byte aligned).
 * want = session when zk_flags == 1 (EPHEMERAL), else 0.  Record i is REGK_DELTA_REPLACE when it is the first record
 * with its path, node j has that path and ephemeral_owner[j] != want - a stale ephemeral of an earlier session (which
 * the server would delete when that session expires), another session's ephemeral, or a persistent node where an
 * ephemeral is wanted (and the reverse).  The payload is not compared then.  Every other class is as in regk_reconcile;
 * the node of a REPLACE record is KEEP (its delete travels inside the replace frame).
 * n_same + n_create + n_update + n_dup + n_replace == n.
 * Edge: a persistent node that has children, where an ephemeral is wanted, is REPLACE too; ZooKeeper then aborts the
 * multi with NOTEMPTY, as the reference's unlink fails there.  An ephemeral node has no children, so the reverse cannot.
 * Refused besides regk_reconcile's refusals (REGK_ERR_INVALID_ARG): stat NULL, an array NULL while m > 0, misaligned
 * device arrays, zk_flags other than 0 or 1 (a sequential or container mode makes a path key meaningless), zk_flags == 1
 * with session == 0.  The delta's arrays are valid until the next regk_reconcile / regk_reconcile_owned call.
 */
typedef struct regk_node_stat {
    const int32_t *version;         /* [m] Stat.version of snapshot node j (passed through verbatim) */
    const int64_t *ephemeral_owner; /* [m] Stat.ephemeralOwner of node j; 0 = persistent */
    int64_t  session;               /* session id the repair will be sent on */
    uint32_t zk_flags;              /* CreateMode of the batch's nodes: 1 = EPHEMERAL, 0 = persistent; nothing else */
    uint32_t reserved;
} regk_node_stat;

#define REGK_DELTA_REPLACE 4u       /* cls[]: only regk_reconcile_owned produces it */

typedef struct regk_delta_owned {
    regk_delta d;                   /* filled as regk_reconcile fills it; cls[] may hold REGK_DELTA_REPLACE */
    uint64_t n_replace;
    const uint64_t *replace;        /* [n_replace] ascending record indices */
} regk_delta_owned;

int         regk_reconcile_owned(regk_ctx *ctx, const regk_decode_in *snapshot, const regk_node_stat *stat,
                                 uint32_t flags, regk_delta_owned *out);

/*
 * ---- the replies to the getData frames of a batch, as a snapshot (the input half of the heartbeat: lib/zk.js:21-44
 * stats every node, lib/index.js:131-159; and of re-registration after a session loss, lib/register.js:85-95,
 * :228-239) -------------------------------------------------------------------------------------------------------------
 * bytes[0, len) = what the caller read off the session after sending the frames of the last REGK_ZK_GETDATA
 * regk_jute_requests call, back to back, from the first reply's length word on; host memory, or device memory with
 * REGK_IN_DEVICE in flags (16-byte aligned).  Frame = int len | ReplyHeader{int xid; long zxid; int err} | body, big
 * endian; body = GetDataResponse{buffer data (D = -1: null, read as empty); Stat (68 bytes)} when err == 0 (len == 88 +
 * max(D, 0)), none otherwise (len == 16).  ZooKeeper answers a session's requests in order: the k-th frame that is not
 * a watch notification (xid -1) or a ping (xid -2) must carry xid == xid_base + k (wrapping) and answers record k.
 * Notifications and pings met before the n-th reply are skipped and counted; the stream may go on past the n-th reply.
 * n_found + n_missing + n_error == n.  err[k] = ReplyHeader.err of record k's reply.
 * snapshot: one node per distinct path among the replies with err == 0 (the first such reply gives it; later ones with
 * the same path are dropped, as regk_reconcile refuses a snapshot that repeats a path; paths are compared byte for byte,
 * a hash only picks a table slot).  Node j = record node_rec[j]: its path from the batch, its data from the reply, its
 * Stat.version and Stat.ephemeralOwner - exactly the input regk_reconcile_owned(ctx, &out->snapshot, {version,
 * ephemeral_owner, session, zk_flags}, ...) takes.  The snapshot holds the batch's own paths only, so a reconcile against
 * it lists no DELETE.  A record whose reply is NONODE (-101) gets no node, so reconcile classes it CREATE; so does a
 * record whose reply carries any other error: do not send the repair while n_error > 0.
 * err and node_rec are pinned host arrays, or device arrays with REGK_OUT_DEVICE; the snapshot, version and
 * ephemeral_owner are always device arrays.  All stay valid until the next regk_read_replies call (a later batch does
 * not touch them).
 * REGK_ERR_STATE: no REGK_ZK_GETDATA framing since the batch finished last, a batch finished since that framing, or a
 * pending batch.  REGK_ERR_INVALID_ARG (the message names the byte position and the expected xid): the stream ends
 * before the n-th reply is complete (and says how many were), len < 16, a negative xid other than -1 / -2, an xid
 * outside the framed range, a reply out of order or for a record that already has one, a success frame whose length
 * disagrees with its data length, D < -1, Stat.dataLength != max(D, 0), an error reply with a body; an xid range
 * [xid_base, xid_base + n) that covers -1 or -2; NULL pointers; a misaligned device stream.
 * PARITY UNPINNED: the reply layout is restated from zookeeper.jute and tested against an independent restatement.
 */
typedef struct regk_replies {
    uint64_t n;                     /* requests: records of the framed batch */
    uint64_t m;                     /* snapshot nodes: one per distinct path among replies with err == 0 */
    uint64_t n_found, n_missing, n_error;   /* replies with err 0 / NONODE (-101) / any other err */
    uint64_t n_skipped;             /* watch notifications (xid -1) and pings (xid -2) met before the n-th reply */
    uint64_t consumed;              /* stream bytes up to the end of the n-th reply */
    uint32_t flags, launches;
    const int32_t  *err;            /* [n] ReplyHeader.err of record i's reply; REGK_OUT_DEVICE decides host/device */
    const uint64_t *node_rec;       /* [m] record whose reply gave node j, ascending; same side as err */
    regk_decode_in  snapshot;       /* ALWAYS device (REGK_IN_DEVICE set): path j = that record's path from the batch,
                                       data j = the reply's data; aligned as regk_reconcile requires */
    const int32_t  *version;        /* [m] device: Stat.version */
    const int64_t  *ephemeral_owner;/* [m] device: Stat.ephemeralOwner */
    float kernel_ms;
} regk_replies;

int         regk_read_replies(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint32_t flags, regk_replies *out);

/*
 * ---- list the batch's service directories and find the instances it no longer produces (the reference removes a node
 * only through its own unregister, lib/register.js:254-295, or through session expiry, which keeps a dead instance in
 * DNS for minutes, README.md:70-76, :764-779) ------------------------------------------------------------------------
 * regk_children_requests, opts->op:
 *   REGK_ZK_GETCHILDREN  one GetChildrenRequest{dir, watch = false} per directory of the batch finished last: frame k =
 *                        len | xid_base + k (wrapping) | 8 | P | dir | 0, 17 + P bytes (the getData layout).  The
 *                        directories are the distinct parent directories of its paths, in order of first record (the
 *                        unique_first order of regk_parent_dirs); directory k = path_{dir_rec[k]}[0, dir_len[k]).  "/"
 *                        is not listed (its children are /zookeeper and every other tree), nor is a directory
 *                        ZooKeeper rejects (regk_mkdirp_dirs' INVALID rule): their first records come back in
 *                        regk_read_children's unlisted[].  A skip-mode batch contributes its kept records.  group != 0
 *                        is REGK_ERR_INVALID_ARG.  REGK_ERR_STATE: a batch of alias nodes (REGK_NODE_ALIAS: an alias
 *                        node's parent is a domain's parent directory, which holds other services - only a host-node
 *                        batch's directories are service directories whose children are that service's instances), no
 *                        finished batch with a path stream (a REGK_NO_PATH batch, an empty batch, a REGK_JOB_STEP
 *                        result), a pending batch.  A successful call records the batch, xid_base, the number of
 *                        directories d and the directory set for regk_read_children; it leaves the REGK_ZK_GETDATA
 *                        record of regk_jute_requests and the results of regk_parent_dirs / regk_mkdirp_dirs as they are.
 *   REGK_ZK_DELETE       DeleteRequest{path, version} for every stale child of the last regk_read_children call
 *                        (REGK_ERR_STATE without one), in stale order; version and group mean what they mean for
 *                        regk_reconcile_requests.  A getChildren reply carries no Stat of a child, so version is
 *                        opts->version (-1 = any).  Built from the library's own copy of the stale paths: neither the
 *                        reply stream nor the batch is needed.
 * Any other op is REGK_ERR_INVALID_ARG.  flags: REGK_OUT_DEVICE returns device pointers, else pinned host arrays; each
 * op's frames are valid until the next call with that op.
 *
 * regk_read_children: bytes[start, len) = what the caller read off the session after sending the getChildren frames,
 * from the first reply's length word on; host memory, or device memory with REGK_IN_DEVICE (bytes 16-byte aligned;
 * start need not be, so the getData replies and these can be one stream: start = regk_replies.consumed).  Every
 * position reported, consumed included, counts from bytes.  Frame = int len | ReplyHeader{int xid; long zxid; int err}
 * | body; body = GetChildrenResponse{int count | count x (int L | L bytes)} iff err == 0 (len == 20 + sum(4 + L_i));
 * count == -1 (a null vector) reads as no children.  Replies come in order: the k-th frame that is not a watch
 * notification (xid -1) or a ping (xid -2) carries xid_base + k and answers directory k; notifications and pings met
 * before the d-th reply are skipped and counted, and the stream may go on past it.
 * Child q of directory k is listing entry child_off[k] + q, in the reply's order.  Listing path e = directory + '/' +
 * name (listing: ALWAYS device, REGK_IN_DEVICE, host_nodes = 1, every entry with empty data - regk_decode reads the
 * instance names back out of it).  cls[e] = REGK_DELTA_KEEP when path e is a path of the batch or a proper ancestor
 * directory of one (a prefix of a listed directory that ends at a component boundary), else REGK_CHILD_STALE; stale[]
 * lists the stale entries ascending.  Names are compared byte for byte (a hash only picks a table slot).  Two equal
 * names in one reply are not looked for, since a server cannot hold them: both get the same class.
 * OWNERSHIP: every child of a listed directory that the batch does not produce is stale, so list only directories
 * whose instances the batch is authoritative for.  A directory whose reply carries an error contributes no children:
 * NONODE (-101) only means it does not exist yet, and the deletes for the other directories stay correct.  Listing is
 * not recursive: a stale child that has children of its own fails its delete with NOTEMPTY.
 * n_found + n_missing + n_error == n_dirs.  dir_rec, dir_len, err, child_off, cls, stale and unlisted are pinned host
 * arrays, or device arrays with REGK_OUT_DEVICE; all results stay valid until the next regk_read_children call (a later
 * batch or framing does not touch them).
 * REGK_ERR_STATE: no REGK_ZK_GETCHILDREN framing, a batch finished since it, a pending batch.  REGK_ERR_INVALID_ARG (the
 * message names the byte position - the frame's, and the entry's for an entry fault - and the expected xid; it is the
 * first fault a front-to-back reader meets): the stream ends before the d-th reply is complete, len < 16, a negative
 * xid other than -1 / -2, an xid outside the framed range, a reply out of order, an error reply with a body, a count
 * below -1, a success frame too short for its count, an entry that runs past its frame, L < 1, a name holding '/' or
 * NUL or equal to "." or "..", entries that end before their frame does; an xid range that covers -1 or -2; d or the
 * number of children not below 2^32 - 1; start > len; NULL pointers; a misaligned device stream.
 * PARITY UNPINNED: the layouts are restated from zookeeper.jute and tested against an independent restatement.
 */
#define REGK_ZK_GETCHILDREN 8u
#define REGK_CHILD_STALE    1u      /* regk_children.cls[]; REGK_DELTA_KEEP (0) otherwise */

int         regk_children_requests(regk_ctx *ctx, const regk_jute_opts *opts, regk_frames *out);

typedef struct regk_children {
    uint64_t n_dirs;                /* d: directories listed */
    uint64_t n_children;            /* listing entries */
    uint64_t n_stale;
    uint64_t n_found, n_missing, n_error;   /* replies with err 0 / NONODE (-101) / any other err */
    uint64_t n_skipped;             /* watch notifications and pings met before the d-th reply */
    uint64_t consumed;              /* stream position of the end of the d-th reply (start when d == 0) */
    uint64_t n_unlisted;
    uint32_t flags, launches;       /* REGK_OUT_DEVICE */
    const uint64_t *dir_rec;        /* [n_dirs] first record of directory k */
    const uint32_t *dir_len;        /* [n_dirs] */
    const int32_t  *err;            /* [n_dirs] ReplyHeader.err of directory k's reply */
    const uint64_t *child_off;      /* [n_dirs + 1] */
    const uint8_t  *cls;            /* [n_children] REGK_DELTA_KEEP / REGK_CHILD_STALE */
    const uint64_t *stale;          /* [n_stale] listing indices, ascending */
    const uint64_t *unlisted;       /* [n_unlisted] first records of "/" and of directories ZooKeeper rejects */
    regk_decode_in  listing;        /* ALWAYS device: path e = directory + '/' + name, empty data */
    float kernel_ms;
} regk_children;

int         regk_read_children(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, uint32_t flags,
                               regk_children *out);

/*
 * ---- the replies to the write frames this library made: each create, delete, setData and replace's outcome, mapped
 * back to what it was framed for (the reference learns each write's outcome from its callback: cleanupPreviousEntries
 * ignores NO_NODE, lib/register.js:88; zkplus' mkdirp ignores NODE_EXISTS) ---------------------------------------------
 * Every successful write framing records what it framed, one record per source (opts->source):
 *   REGK_RES_BATCH      the last regk_jute_frames, or regk_jute_requests with REGK_ZK_CREATE / _DELETE / _SETDATA (a
 *                       REGK_ZK_GETDATA framing does not replace it); entry e = record e of the batch finished last
 *   REGK_RES_MKDIRP     the last regk_mkdirp_requests; entry k = directory k of the mkdirp set
 *   REGK_RES_RECONCILE  the last regk_reconcile_requests with opts->op (REGK_ZK_CREATE, _DELETE, _SETDATA or
 *                       REGK_ZK_REPLACE: one record each, so the whole repair can be framed before anything is sent);
 *                       entry e = list entry e
 *   REGK_RES_STALE      the last regk_children_requests(REGK_ZK_DELETE); entry e = stale entry e
 * The record holds the xid base, the frame count, the group (a replace frame holds max(g, 1) entries of two operations)
 * and the entry count; the paths stay where the library keeps them (the batch's path stream, the mkdirp set, the
 * reconcile's gathered streams, the packed stale paths).  REGK_ERR_STATE: no such framing, or the state it framed has
 * changed since - a batch finished (BATCH), regk_mkdirp_dirs ran (MKDIRP), a reconcile ran (RECONCILE),
 * regk_read_children ran (STALE) - or a pending batch.
 * bytes[start, len) = what the caller read off the session after sending those frames, from the first reply's length
 * word on; host memory, or device memory with REGK_IN_DEVICE in opts->flags (16-byte aligned; start need not be, so one
 * stream can hold the replies of several sections: start = the previous section's consumed).  Positions count from
 * bytes.  The k-th frame that is not a watch notification (xid -1) or a ping (xid -2) must carry xid_base + k and answers
 * frame k; notifications and pings before the last reply are skipped and counted.
 * Reply layouts (zookeeper.jute; big endian; frame = int len | ReplyHeader{int xid; long zxid; int err} | body):
 *   create   err == 0: CreateResponse{path}, len == 20 + P; the path must equal the framed path byte for byte
 *   delete   len == 16
 *   setData  err == 0: Stat, len == 84; Stat.dataLength must equal the framed data's length; version[e] = Stat.version
 *   error    err != 0: len == 16, no body; in a multi frame every operation then fails with err
 *   multi    err == 0: MultiResponse, one MultiHeader{type, done = 0, err} + result per operation, then
 *            MultiHeader{-1, 1, -1}.  Applied: typed results (type = the framed op; create 4 + P bytes of path, delete
 *            none, setData a 68-byte Stat).  Rolled back: only ErrorResults (MultiHeader{-1, 0, e} ErrorResponse{e}, 13
 *            bytes each): 0 before the failing operation, its code, then -2 (RUNTIMEINCONSISTENCY).
 * Since a multi reply is all typed results or all ErrorResults and every framed path length is known, each entry's result
 * position is closed form: frame + 20 + a prefix of the frame's result sizes (applied), frame + 20 + 13 x the operation
 * index (rolled back).  cls[e]:
 *   REGK_RES_DONE     the write took effect; also a delete answered NONODE (-101) and a mkdirp create answered
 *                     NODEEXISTS (-110), the reference's two tolerances, with that code kept in err[e]
 *   REGK_RES_FAILED   the entry's own operation failed (an error reply, the failing operation of a rolled-back multi, or
 *                     any operation of a multi answered with a header error); err[e] is its code
 *   REGK_RES_ABORTED  another entry's failure rolled its multi transaction back; err[e] is its operations' first nonzero
 *                     code (-2 after the failing one), else 0
 * version[e] = the new Stat.version of a setData that took effect, 0 for a create or replace that took effect, else -1.
 * subject[e] = the record (BATCH; RECONCILE create, setData, replace), the snapshot node (RECONCILE delete), the directory
 * (MKDIRP) or the listing entry (STALE) the entry was framed for.  failed[] / aborted[] list the FAILED / ABORTED entries
 * ascending.  n_done + n_failed + n_aborted == n_entries.  The arrays are pinned host arrays, or device arrays with
 * REGK_OUT_DEVICE; all stay valid until the next regk_read_results call.
 * REGK_ERR_INVALID_ARG (the message names the byte position, that of the frame and of the entry, and the expected xid; it
 * is the first fault a front-to-back reader meets): the stream ends before the last reply is complete, len < 16, a
 * negative xid other than -1 / -2, an xid outside the framed range, a reply out of order, an error reply with a body, a
 * success length that fits neither outcome of its frame, a MultiHeader of the wrong type, done flag or err, a missing
 * closing MultiHeader, a create path echo that differs from the framed path, a Stat.dataLength that differs from the
 * framed data, an ErrorResult whose two codes differ or that breaks the 0 / code / -2 order, a rolled-back multi with no
 * nonzero ErrorResult; an xid range that covers -1 or -2; a source or op not listed above; start > len; NULL pointers; a
 * misaligned device stream.
 * PARITY UNPINNED: the layouts are restated from zookeeper.jute and the server's multi handling, and tested against an
 * independent restatement, not against a server.
 */
#define REGK_RES_BATCH      1u
#define REGK_RES_MKDIRP     2u
#define REGK_RES_RECONCILE  3u
#define REGK_RES_STALE      4u

#define REGK_RES_DONE    0u         /* regk_results.cls[] */
#define REGK_RES_FAILED  1u
#define REGK_RES_ABORTED 2u

typedef struct regk_results_opts {
    uint32_t source;                /* REGK_RES_* */
    uint32_t op;                    /* REGK_RES_RECONCILE: REGK_ZK_CREATE / _DELETE / _SETDATA / REGK_ZK_REPLACE */
    uint32_t flags;                 /* REGK_IN_DEVICE | REGK_OUT_DEVICE */
    uint32_t reserved;
} regk_results_opts;

typedef struct regk_results {
    uint64_t n_frames, n_entries;
    uint64_t n_done, n_failed, n_aborted;
    uint64_t n_skipped;             /* watch notifications and pings met before the last reply */
    uint64_t consumed;              /* stream position of the end of the last reply (start when there are no frames) */
    uint32_t flags, launches;       /* REGK_OUT_DEVICE */
    const int32_t  *frame_err;      /* [n_frames] ReplyHeader.err of frame k's reply */
    const int32_t  *err;            /* [n_entries] */
    const uint8_t  *cls;            /* [n_entries] REGK_RES_DONE / _FAILED / _ABORTED */
    const int32_t  *version;        /* [n_entries] */
    const uint64_t *subject;        /* [n_entries] */
    const uint64_t *failed;         /* [n_failed] entry indices, ascending */
    const uint64_t *aborted;        /* [n_aborted] */
    float kernel_ms;
} regk_results;

int         regk_read_results(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start,
                              const regk_results_opts *opts, regk_results *out);

/*
 * ---- the heartbeat by stat: an exists per node, the replies read and the batch classed without any node data (the
 * reference's heartbeat is zk.stat on every node, lib/zk.js:21-44: one ExistsRequest out and a 68-byte Stat back) ------
 * regk_read_stats: bytes[start, len) = what the caller read off the session after sending the frames of the last
 * REGK_ZK_EXISTS regk_jute_requests call, from the first reply's length word on; host memory, or device memory with
 * REGK_IN_DEVICE (bytes 16-byte aligned; start need not be, so the replies can follow other sections in one stream).
 * Positions, consumed included, count from bytes.  Frame = int len | ReplyHeader{int xid; long zxid; int err} | body, big
 * endian; body = ExistsResponse{Stat (68 bytes)} iff err == 0, so len == 84 for a success and 16 otherwise.  Stat =
 * czxid mzxid ctime mtime (8 each) | version cversion aversion (4 each) | ephemeralOwner (8) | dataLength numChildren (4
 * each) | pzxid (8).  The k-th frame that is not a watch notification (xid -1) or a ping (xid -2) must carry xid_base + k
 * (wrapping) and answers record k; notifications and pings met before the n-th reply are skipped and counted, and the
 * stream may go on past it.  n_found + n_missing + n_error == n; the registry is healthy iff n_missing + n_error == 0,
 * which is all the reference's heartbeat asks.
 * err[k] = ReplyHeader.err; version, ephemeral_owner, data_length and mzxid are record k's Stat fields, 0 where err[k] !=
 * 0.  The five arrays are pinned host arrays, or device arrays with REGK_OUT_DEVICE; the library keeps its device copies
 * for regk_reconcile_stats either way.  All stay valid until the next regk_read_stats call; a later batch does not free
 * them, but regk_reconcile_stats then refuses them.
 * REGK_ERR_STATE: no REGK_ZK_EXISTS framing since the batch finished last, a batch finished since that framing, or a
 * pending batch.  REGK_ERR_INVALID_ARG (the message names the byte position and the expected xid; it is the first fault
 * a front-to-back reader meets): the stream ends before the n-th reply is complete (and says how many were), len < 16, a
 * negative xid other than -1 / -2, an xid outside the framed range, a reply out of order or for a record that already
 * has one, an error reply with a body, a success length other than 84, Stat.dataLength < 0; an xid range that covers -1
 * or -2; start > len; NULL pointers; a misaligned device stream.
 * PARITY UNPINNED: the layout is restated from zookeeper.jute and tested against an independent restatement.
 */
typedef struct regk_stats {
    uint64_t n;                     /* requests: records of the framed batch */
    uint64_t n_found, n_missing, n_error;   /* replies with err 0 / NONODE (-101) / any other err */
    uint64_t n_skipped;             /* watch notifications and pings met before the n-th reply */
    uint64_t consumed;              /* stream position of the end of the n-th reply */
    uint32_t flags, launches;       /* REGK_OUT_DEVICE */
    const int32_t *err;             /* [n] ReplyHeader.err of record k's reply */
    const int32_t *version;         /* [n] Stat.version */
    const int64_t *ephemeral_owner; /* [n] Stat.ephemeralOwner; 0 = persistent */
    const int32_t *data_length;     /* [n] Stat.dataLength */
    const int64_t *mzxid;           /* [n] Stat.mzxid: the zxid of the node's last write */
    float kernel_ms;
} regk_stats;

int         regk_read_stats(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, uint32_t flags,
                            regk_stats *out);

/*
 * regk_reconcile_stats: class the batch finished last from the stats of the last regk_read_stats call, and leave the
 * context as regk_reconcile_owned leaves it: the lists, each update / replace entry's observed version and the gathered
 * request streams, so regk_reconcile_requests (create / setData / replace, REGK_ZK_VERSION_OBSERVED, groups) and
 * regk_read_results(REGK_RES_RECONCILE) follow unchanged.  Reply k answers record k, so there is no snapshot and no
 * observed side: m == 0, n_delete == 0, obs_cls == NULL, and REGK_ZK_DELETE frames nothing (nodes the batch does not
 * produce are regk_read_children's business).  want = session when zk_flags == 1 (EPHEMERAL), else 0.  Record i:
 *   REGK_DELTA_DUP      an earlier record has the same path (compared byte for byte; the first occurrence decides)
 *   REGK_DELTA_CREATE   its reply is NONODE
 *   REGK_DELTA_REPLACE  found, and ephemeral_owner[i] != want; nothing else is looked at
 *   REGK_DELTA_UPDATE   found, the owner is right, and data_length[i] differs from payload i's length - or known_mzxid
 *                       is given and mzxid[i] != known_mzxid[i]
 *   REGK_DELTA_SAME     otherwise
 * match[i] = the first record with path i, or UINT64_MAX when that record's node is missing.
 * n_same + n_create + n_update + n_dup + n_replace == n.
 * WHAT A STAT CANNOT SEE: a node whose bytes changed to a payload of the same length (an address rewritten from 10.0.0.1
 * to 10.0.0.2) is SAME unless known_mzxid is given.  known_mzxid[i] = the mzxid record i's node had when its bytes were
 * last verified (a getData round whose regk_reconcile_owned said SAME, with the regk_read_stats of the same round sent
 * first; INTEGRATION.md §3): any write since then moves mzxid and makes the record UPDATE.  NULL, or int64[n]: a host
 * array, or a device array (8-byte aligned) with REGK_IN_DEVICE in flags.  flags: REGK_OUT_DEVICE as regk_reconcile.
 * REGK_ERR_STATE: no regk_read_stats result, a batch finished since it, a pending batch; or a reply with an error other
 * than NONODE - the message names the smallest such record and its code: a repair built over an unknown node state is
 * never right.  REGK_ERR_INVALID_ARG: zk_flags other than 0 or 1, zk_flags == 1 with session == 0, a misaligned device
 * known_mzxid, NULL pointers.  The delta's arrays are valid until the next reconcile call of any kind.
 */
typedef struct regk_stat_opts {
    int64_t  session;               /* session id the repair will be sent on */
    uint32_t zk_flags;              /* CreateMode of the batch's nodes: 1 = EPHEMERAL, 0 = persistent; nothing else */
    uint32_t reserved;
    const int64_t *known_mzxid;     /* [n] or NULL */
} regk_stat_opts;

int         regk_reconcile_stats(regk_ctx *ctx, const regk_stat_opts *opts, uint32_t flags, regk_delta_owned *out);

/*
 * ---- the watched heartbeat: arm each node and service directory once (REGK_ZK_WATCH), read the notifications the
 * server pushes for what changed, and re-check and re-arm only that.  An additional route: the reference polls every
 * node with zk.stat (lib/zk.js:21-44), and the stat round above stays as it is ----------------------------------------
 * regk_read_events: bytes[start, len) = what the caller read off the session; host memory, or device memory with
 * REGK_IN_DEVICE in opts->flags (bytes 16-byte aligned; start need not be).  Positions, consumed included, count from
 * bytes.  Every complete frame from start on is walked:
 *   notification  int len | ReplyHeader{int xid = -1; long zxid; int err = 0} | WatcherEvent{int type; int state;
 *                 ustring path}, so len == 28 + P (P = the path's length word, the path at +32 from the frame's first
 *                 byte).  The header's zxid is reported, not checked: server versions differ in what they put there.
 *   ping          xid -2, len == 16.
 *   reply         an xid in [opts->xid_base, opts->xid_base + opts->n_xids) (wrapping): a reply to an outstanding
 *                 request, skipped by its length whatever its body and counted, so one session stream can go through
 *                 this call and through the reply readers, each reading its own frames and skipping the other's.
 * A trailing partial frame is not an error (a socket read can end mid-frame): consumed stops at its start and
 * out->partial = 1; feed the rest with the next call.  Without one, consumed == len.
 * Event e (in stream order) has pos, type, state, zxid and a subject, mapped by the event's path (compared byte for byte;
 * a hash only picks a table slot):
 *   NodeCreated (1), NodeDeleted (2), NodeDataChanged (3)  the first record of the batch finished last with that path
 *                                                          (REGK_EV_RECORD; a DUP record is never a subject itself)
 *   NodeChildrenChanged (4), and NodeDeleted (2) of a path that is no record's
 *                                                          service directory k of the batch, in the order and by the
 *                                                          rule regk_children_requests lists them (REGK_EV_DIR)
 *   anything else, or a path in neither set               REGK_EV_NONE, subject UINT64_MAX
 * n_unmatched counts the REGK_EV_NONE events; n_other counts types -1 and 5 .. 7 (session events and watch removals),
 * which are also unmatched.  Each mapped record event ORs its type's bit into its record's mark and each directory event
 * marks its directory; a record or directory not yet pending joins the pending set, which accumulates over the calls of
 * one batch generation (feed each recv separately) until regk_events_requests takes it.  A new batch drops it.  The
 * tables are built on the first call after a batch finishes (work proportional to n); every later call's work is
 * proportional to its stream and its events.  n_dirty_recs / n_dirty_dirs = what is pending after the call.
 * pos .. subject are pinned host arrays, or device arrays with REGK_OUT_DEVICE; valid until the next call.
 * REGK_ERR_STATE: no finished batch with a path stream, a pending batch.  REGK_ERR_INVALID_ARG (the message names the
 * byte position; nothing is marked): len < 16, an xid other than -1 / -2 outside the reply range, a notification whose
 * length is not 28 + P, P < 0, a notification with err != 0 or a type outside -1 .. 7, a ping with a body; a reply range
 * that covers -1 or -2; start > len; NULL pointers; a misaligned device stream.
 *
 * regk_events_requests: frame the pending set of op, in ascending order, and clear it.  Watches are one-shot, so every
 * frame carries watch = 1 whatever opts->flags says (only REGK_OUT_DEVICE is read from it); group must be 0.
 *   REGK_ZK_EXISTS       one ExistsRequest per pending record (an exists watch arms a missing node as well as a present
 *                        one).  Recorded as a SUBSET exists framing: regk_read_stats reads its replies unchanged, reply k
 *                        answering pending record k and its arrays holding one entry per pending record; then
 *                        regk_reconcile_stats classes the whole batch: a pending record by its stat, as always, every
 *                        other record SAME (its watch has not fired), DUP detection over all n.  known_mzxid with a
 *                        subset is REGK_ERR_INVALID_ARG: the repair's own writes fire the library's watches and move
 *                        mzxid, so an mzxid baseline would never settle.  What a stat cannot see stays unseen: a
 *                        same-length rewrite still fires NodeDataChanged, and the re-check then reads it as SAME.
 *   REGK_ZK_GETCHILDREN  one GetChildrenRequest per pending directory, recorded as the last getChildren framing:
 *                        regk_read_children reads it unchanged over that subset (dir_rec / dir_len are the subset's,
 *                        n_unlisted == 0, the keep table still holds every directory of the batch), and
 *                        regk_children_requests(REGK_ZK_DELETE) frames the stale children it finds.
 * An empty pending set frames 0 requests and succeeds.  Any other op, group != 0: REGK_ERR_INVALID_ARG.  No
 * regk_read_events call since the batch finished last, a pending batch, an exists framing of a batch without its payload
 * stream: REGK_ERR_STATE.  flags: REGK_OUT_DEVICE as regk_jute_requests; the frames stay valid until the next call with
 * that op.
 * CONVERGENCE: the repair's own writes fire the library's own watches, so the next regk_read_events makes those records
 * dirty; their re-check says SAME and re-arms them (a replaced node included).  Every byte the session delivers must pass
 * through regk_read_events once.  After a reconnect, regk_setwatches_requests below carries the watches over; after a
 * session expiry, run the full armed round again (the read framings with REGK_ZK_WATCH).
 * PARITY UNPINNED: the layouts are restated from zookeeper.jute (ReplyHeader, WatcherEvent, ExistsRequest,
 * GetChildrenRequest) and tested against an independent restatement, not against a server.
 */
#define REGK_EV_NONE    0u          /* regk_events.subject_kind[] */
#define REGK_EV_RECORD  1u
#define REGK_EV_DIR     2u

typedef struct regk_events_opts {
    int32_t  xid_base;              /* the replies still outstanding on the session: [xid_base, xid_base + n_xids) */
    uint32_t n_xids;
    uint32_t flags;                 /* REGK_IN_DEVICE | REGK_OUT_DEVICE */
    uint32_t reserved;
} regk_events_opts;

typedef struct regk_events {
    uint64_t n_events, n_pings, n_replies;
    uint64_t n_unmatched, n_other;
    uint64_t consumed;              /* end of the last complete frame (start when none) */
    uint64_t n_dirty_recs, n_dirty_dirs;    /* pending after the call */
    uint32_t partial;               /* 1: a frame starts at consumed and the stream ends inside it */
    uint32_t flags, launches;       /* REGK_OUT_DEVICE */
    uint32_t reserved;
    const uint64_t *pos;            /* [n_events] the frame's first byte */
    const int32_t  *type;           /* WatcherEvent.type */
    const int32_t  *state;          /* WatcherEvent.state */
    const int64_t  *zxid;           /* ReplyHeader.zxid */
    const uint8_t  *subject_kind;   /* REGK_EV_* */
    const uint64_t *subject;        /* record, directory, or UINT64_MAX */
    float kernel_ms;
} regk_events;

int         regk_read_events(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, const regk_events_opts *opts,
                             regk_events *out);
int         regk_events_requests(regk_ctx *ctx, const regk_jute_opts *opts, regk_frames *out);

/*
 * ---- the watched heartbeat across a reconnect: ZooKeeper forgets a connection's watches when it drops, though the
 * session survives.  regk_setwatches_requests frames SetWatches (op 101) for the watches the session holds, so the
 * server re-arms them on the new connection or fires what the client missed, and re-pends everything else -----------
 * The context keeps, per batch generation, the watch kind each first-of-path record and each service directory holds:
 *   regk_read_stats of an exists framing with the watch byte (REGK_ZK_WATCH, or an regk_events_requests subset): err 0
 *   gives DATA, NONODE gives EXIST (an exists watch arms a missing node too), any other err NONE.
 *   regk_read_children of a getChildren framing with the watch byte: err 0 gives CHILD, anything else NONE (ZooKeeper
 *   leaves no child watch on a missing node).
 * Unwatched reads leave the kinds alone; a new batch resets them all to NONE.  A watched framing whose replies have not
 * been read is in flight: its requests die with the connection, so its items count as NONE.  The bookkeeping after a
 * watched read is one kernel that the read's `launches` and kernel_ms do not include.
 * The session zxid is the largest ReplyHeader.zxid of every complete reply a successful regk_read_events call walked
 * (replies in the outstanding xid range and SetWatches replies; not notifications or pings), 0 at first, kept for the
 * context's whole life.  It is safe as relativeZxid: a reply with zxid R leaves the server after every notification of
 * a change at or below R, and TCP keeps that order, so an event the client missed is one the session never delivered,
 * and then R was not read either.  Underestimating is always safe: the server only fires spurious events, which cost
 * re-checks.
 *
 * regk_setwatches_requests: call it when the connection drops, before reconnecting; relative_zxid is also the
 * lastZxidSeen of the ConnectRequest.  The lists, each without the pending records and directories (their re-check
 * re-arms them):
 *   D  the records of kind DATA, ascending          E  the records of kind EXIST, ascending
 *   C  the directories of kind CHILD, in the order regk_children_requests lists them
 * Every other first-of-path record and every other directory joins the current pending set (NONE, in flight, never
 * armed; n_repend_*), so after the call each one is either listed or pending and regk_events_requests re-checks the
 * rest.  With no watched round read, nothing is listed and everything is pending.
 * Frames, big endian: int len | int xid = -8 | int type = 101 | long relativeZxid | int nD | nD x (int P | path) | int nE
 * | ... | int nC | ..., 32 bytes of header and count words each.  The split, in closed form: with S = D ++ E ++ C, s_j the
 * exclusive prefix of the entry sizes 4 + P, Lmax = 4 + the batch's longest path and B = max_frame - 32 - Lmax, entry j
 * goes into frame floor(s_j / B).  Every frame holds at least one entry and is shorter than max_frame (len + 4 bytes).
 * max_frame 0 means 131072 (the Java client's 128 KiB); below 32 + 2 Lmax, or 2^31 or more, it is refused (the message
 * names the minimum).  The server closes the connection when a frame's len exceeds its jute.maxbuffer (1048575 by
 * default).  frames.frame_bytes / frame_off are pinned host arrays, or device arrays with REGK_OUT_DEVICE in
 * opts->flags; valid until the next call.  Empty lists frame 0 frames.
 * After a successful call regk_read_events, for this batch generation, also accepts a SetWatches reply (xid -8, len 16,
 * err 0: skipped and counted in n_replies, its zxid entering the high-water mark); a -8 frame with a body or an err is
 * refused.  Without the call, -8 is refused as any negative xid.
 * REGK_ERR_STATE: a pending batch, no finished batch with a path stream.  REGK_ERR_INVALID_ARG: NULL pointers, a bad
 * max_frame, unknown flag bits.  The tables are built on demand, as regk_read_events builds them.
 * PARITY UNPINNED: the layout is restated from zookeeper.jute (SetWatches) and the server's re-arming from ZooKeeper
 * 3.4's DataTree.setWatches, tested against an independent restatement, not against a server.
 */
typedef struct regk_setwatches_opts {
    uint32_t max_frame;             /* bytes per frame, len word included; 0 = 131072 */
    uint32_t flags;                 /* REGK_OUT_DEVICE */
} regk_setwatches_opts;

typedef struct regk_setwatches {
    uint64_t n_data, n_exist, n_child;          /* paths listed */
    uint64_t n_repend_recs, n_repend_dirs;      /* made pending by this call */
    uint64_t n_dirty_recs, n_dirty_dirs;        /* pending after the call, as regk_read_events reports them */
    int64_t  relative_zxid;
    regk_frames frames;
} regk_setwatches;

int         regk_setwatches_requests(regk_ctx *ctx, const regk_setwatches_opts *opts, regk_setwatches *out);

/*
 * ---- what DNS answers for a registry snapshot: the A and SRV sets its host and service records define (the contract
 * between registrar and Binder, README.md:441-755 of the reference), restricted to the canonical forms this library
 * writes ------------------------------------------------------------------------------------------------------------
 * Snapshot: m nodes in the layout regk_reconcile takes (host streams, or device streams with REGK_IN_DEVICE, e.g.
 * regk_replies.snapshot as it stands); host_nodes is ignored; REGK_DECODE_LAST, unknown opts->flags bits, a nonzero
 * reserved, a negative default TTL and m >= 2^32 - 1 are REGK_ERR_INVALID_ARG.  A device snapshot's offsets are checked
 * as regk_reconcile checks them, and two nodes with one path are refused as there (the message names the later node).
 *   name(j)   node j's path components reversed and joined by '.' (regk_decode's domain with host_nodes = 0):
 *             /us/joyent/example/b44c74d6 -> b44c74d6.example.joyent.us.  Valid: every label 1-63 bytes of
 *             [A-Za-z0-9_-], at most 253 bytes.  A service record's SRV owner <srvce>.<proto>.name(s) (srvce and proto
 *             verbatim, README.md:432) must be valid too.
 *   node_cls  the first failing rule decides, in the order of REGK_RSV_* below.  Type tables (README.md:274-282,
 *             type bytes compared raw): queryable db_host host load_balancer moray_host redis_host; usable for a
 *             service load_balancer moray_host ops_host redis_host rr_host.
 *   children  a host record c of class OK and a usable type is a child of service node s when dirname(path(c)) is
 *             s's path byte for byte and s is a service record of class OK; children in ascending node order.
 *   TTLs      a_ttl(c) = c's ttl, else default_host_ttl; srv_ttl(s) = s's service.service.ttl, else default_srv_ttl
 *             (README.md:670-755; in canonical form only the innermost ttl exists).
 * Queries, in ascending node order (a service's A query before its SRV query):
 *   REGK_Q_HOST_A       every OK host record of a queryable type: name(c). a_ttl(c) IN A addr(c)
 *   REGK_Q_SERVICE_A    every OK service record, with or without children: per child
 *                       name(s). min(srv_ttl(s), a_ttl(c)) IN A addr(c)
 *   REGK_Q_SERVICE_SRV  per child, per port of its ports in payload order ([port(s)] without a ports key):
 *                       <srvce>.<proto>.name(s). srv_ttl(s) IN SRV 0 10 port name(c).  (README.md:432,705); additional:
 *                       per child with >= 1 SRV answer, name(c). a_ttl(c) IN A addr(c).  ports: [] gives neither.
 * Text: one record per line, LF-terminated; owner, TTL, IN, type and rdata separated by one TAB, SRV rdata fields by
 * one space: dig's presentation format with single tabs.
 * Results are pinned host arrays, or device arrays with REGK_OUT_DEVICE; valid until the next regk_resolve call.
 * launches counts the radix sort that groups the children as one; kernel_ms spans every pass but the host's reads.
 * PARITY UNPINNED: Binder's default TTLs are parameters (the README's SRV example implies a host default of 30:
 * README.md:383-392 sets no ttl and :433 shows 30); Binder's answer order; a service record with a middle-level ttl
 * (the README's authcache example, :511-523) is not a form this library writes and is REGK_RSV_NOT_RECORD here
 * unless REGK_RESOLVE_ANY_FORM is set.
 *
 * ---- with REGK_RESOLVE_ANY_FORM (regk_resolve and regk_walk_resolve): records in any JSON form Binder reads.  Without
 * the flag nothing changes (the same kernels, launches and bytes).  With it:
 *   1. The canonical recogniser still decides first: every node it accepts keeps exactly its class, record and
 *      answers.  The general reader decides the CANDIDATES only: nodes with non-empty data and a path ('/' first) that
 *      the canonical recogniser classes REGK_RSV_NOT_RECORD.
 *   2. A candidate is REGK_RSV_NOT_RECORD unless its payload is exactly one JSON object (RFC 8259), optionally
 *      surrounded by JSON whitespace (space, TAB, LF, CR); with at most 64 containers nested; bytes >= 0x80 only inside
 *      strings (not validated as UTF-8); and no member name anywhere holding a backslash (an escaped name could decode
 *      to "ttl"; names are compared raw).  Duplicate member names: the last one wins, as in JSON.parse.  String values
 *      are taken verbatim, escapes left as they are (so an escaped type, address or srvce fails the rules below:
 *      UNKNOWN_TYPE, BAD_ADDRESS, BAD_NAME).  Unknown members at any depth are skipped (and grammar-checked).
 *   3. Service record: the top-level "type" is the string "service"; top.service is an object; top.service.service is
 *      an object with "srvce" (a string), "proto" (a string) and "port" (an integer 0..2^32-1); the middle object's
 *      "type" is not required.  srv_ttl = the first present of service.service.ttl, service.ttl, ttl.
 *   4. Host record: the top-level "type" is a string other than "service".  inner = the top-level member whose name
 *      equals the type bytes raw (before or after "type"), an object; inner.address, a string, is the address; the
 *      top-level "address" is ignored (absent, different or of any type); inner.ports is optional, and if present an
 *      array of integers 0..2^32-1 ([] allowed).  a_ttl = the first present of inner.ttl and the top-level ttl.
 *   5. Every "ttl" member of the inspected objects (top, service and service.service of a service record; top and
 *      inner of a host record), the port and each ports element is a JSON integer -?(0|[1-9][0-9]*): no fraction, no
 *      exponent, not -0; a ttl fits in int32.  Anything else there (null, a string, 30.0, ...) is REGK_RSV_NOT_RECORD.
 *      Numbers in skipped members may take any JSON form.
 *   6. From there on everything is as without the flag: BAD_NAME, UNKNOWN_TYPE, BAD_ADDRESS, BAD_TTL (on the chosen
 *      TTL), BAD_PORT, the children, the queries, the text, regk_dns_answer (REGK_DNS_PTR included) and the walk's
 *      identity rules.
 *   7. regk_walk_resolve: a call whose REGK_RESOLVE_ANY_FORM differs from the last successful call's is full, as a
 *      change of default TTLs is.
 *   8. launches counts 2 more kernels (candidate count and compaction), and 1 more (the reader) when there is at least
 *      one candidate; the flag's classify replaces the plain one.
 * PARITY UNPINNED (Binder is absent): Binder's handling of escaped member names, of non-integer or null TTLs and
 * ports, and of a host record without an inner address but with a top-level one; its nesting limit; whether it
 * compares the type value decoded.
 */
#define REGK_RESOLVE_ANY_FORM (1u << 12)    /* regk_resolve_opts.flags: read records in any JSON form (above) */

typedef struct regk_resolve_opts {
    uint32_t flags;                 /* REGK_OUT_DEVICE | REGK_RESOLVE_ANY_FORM */
    int32_t  default_host_ttl;      /* A TTL of a host record without "ttl" (>= 0) */
    int32_t  default_srv_ttl;       /* SRV TTL of a service record without "ttl" (>= 0) */
    uint32_t reserved;              /* 0 */
} regk_resolve_opts;

#define REGK_Q_HOST_A      1u       /* A    <name of node>                 */
#define REGK_Q_SERVICE_A   2u       /* A    <name of service node>         */
#define REGK_Q_SERVICE_SRV 3u       /* SRV  <srvce>.<proto>.<service name> */

#define REGK_RSV_OK           0u    /* node_cls[]; first failing rule decides, in this order: */
#define REGK_RSV_EMPTY        1u    /* empty data: a directory node; answers nothing; not listed */
#define REGK_RSV_NOT_RECORD   2u    /* regk_decode found no canonical host or service record (nor, with
                                       REGK_RESOLVE_ANY_FORM, the general reader any record), or a bad path */
#define REGK_RSV_BAD_NAME     3u    /* a DNS name it would own is not a valid name */
#define REGK_RSV_UNKNOWN_TYPE 4u    /* host record whose type bytes are not one of the README's seven */
#define REGK_RSV_BAD_ADDRESS  5u    /* host record address not a dotted-quad IPv4 (no leading zeros) */
#define REGK_RSV_BAD_TTL      6u    /* ttl < 0 */
#define REGK_RSV_BAD_PORT     7u    /* a port > 65535 (host ports, or the service's port) */

typedef struct regk_answers {
    uint64_t m;                     /* snapshot nodes */
    uint64_t n_queries, n_answers, n_additional, n_unresolved;
    uint64_t text_total;
    uint32_t flags, launches;
    const uint8_t  *q_kind;         /* [n_queries] REGK_Q_* */
    const uint64_t *q_node;         /* [n_queries] snapshot node whose name is asked, ascending */
    const uint64_t *sec_off;        /* [2 n_queries + 1]: answer section of q = text[sec_off[2q], sec_off[2q+1]),
                                       additional section = text[sec_off[2q+1], sec_off[2q+2]) */
    const uint8_t  *text;           /* [text_total] */
    const uint8_t  *node_cls;       /* [m] REGK_RSV_* */
    const uint64_t *unresolved;     /* [n_unresolved] ascending nodes with class >= REGK_RSV_NOT_RECORD */
    float kernel_ms;
} regk_answers;

int         regk_resolve(regk_ctx *ctx, const regk_decode_in *snapshot, const regk_resolve_opts *opts, regk_answers *out);

/*
 * ---- DNS responses from the last regk_resolve: RFC 1035 query messages in, wire-format A and SRV responses out ------
 * Answers against the last regk_resolve (or regk_walk_resolve, below) on the context; REGK_ERR_STATE when there was
 * none or it failed, or when the walk's snapshot changed since that regk_walk_resolve.  A device
 * snapshot passed to that resolve must stay allocated and unchanged until the last regk_dns_answer on it (a host
 * snapshot was staged by the resolve).  Results stay valid until the next regk_dns_answer or regk_resolve.
 * Input: k messages back to back, no TCP length prefix; message i = msgs[off[i], off[i+1]).  Host memory, or device
 * memory with REGK_IN_DEVICE (off 8-byte aligned, total = off[k]).  REGK_ERR_INVALID_ARG: a NULL pointer, unknown flag
 * bits, a nonzero reserved, udp_payload outside 512..65535, misaligned device offsets, offsets that are not monotone
 * or reach past total, a message longer than 65535 bytes; the message names the smallest bad message (device offsets
 * are checked on the device before any message byte is read).
 * Message handling, the first rule that applies decides:
 *   1. shorter than 12 bytes, or QR = 1: REGK_DNS_DROPPED, no response bytes
 *   2. opcode != 0: NOTIMP
 *   3. QDCOUNT != 1, ANCOUNT != 0, NSCOUNT != 0 or ARCOUNT > 1: FORMERR
 *   4. the question must parse, else FORMERR: labels of 1-63 bytes (a length byte with either top bit set, a
 *      compression pointer or an extended label type, is FORMERR), a wire name of at most 255 bytes, QTYPE and QCLASS
 *      inside the message
 *   5. ARCOUNT = 1: an OPT record (root owner, TYPE 41, RDATA inside the message), else FORMERR; its CLASS is the
 *      requester's UDP size, its TTL ext-rcode, version and flags; options are ignored
 *   6. bytes after the last record: FORMERR
 *   7. OPT version != 0: BADVERS (extended rcode 1 in the response OPT, header rcode 0)
 *   8. QCLASS != IN: REFUSED
 *   9. lookup.  Names compare after ASCII lower-casing; a name with a label byte outside [A-Za-z0-9_-], or the root,
 *      owns nothing.  node(name) = the snapshot node whose path is '/' + the lower-cased labels reversed, joined by
 *      '/' (a node whose path has an upper-case letter is the node of no name).  A name owns A when node(name) has a
 *      REGK_Q_HOST_A or REGK_Q_SERVICE_A query; it owns SRV when it has >= 3 labels and node(name without its first
 *      two labels) is a class-OK service record whose srvce and proto equal those two labels, case-insensitively.
 *      QTYPE A on an A owner, QTYPE SRV (33) on an SRV owner: ANSWER with that regk_resolve query's answers (and, for
 *      SRV, additionals); any other QTYPE on a name that owns A or SRV: NODATA; otherwise NXDOMAIN.  A service without
 *      children answers A with NOERROR and no RRs.  node[i] is the answering node for ANSWER, else ~0.
 * Response: ID copied, QR = 1, opcode and RD copied, RA Z AD CD 0, AA = 1 for ANSWER, NODATA and NXDOMAIN.  NOTIMP and
 * FORMERR: the 12-byte header only, QDCOUNT 0.  Every other response echoes the question byte for byte and, when the
 * query had OPT, ends with an OPT record: root owner, TYPE 41, CLASS udp_payload, TTL ext-rcode << 24 | the query's
 * DO bit, RDLENGTH 0.  RRs in the order and with the TTLs of the matching regk_resolve query, ports in payload order:
 *   A      owner 0xC00C, 16 bytes
 *   SRV    owner 0xC00C, priority 0, weight 10, port, the child's name uncompressed (RFC 2782): 20 + L bytes for a
 *          name of L text bytes
 *   additional A of a child: owner a pointer to the target name in the child's first SRV RR (RR start + 18), 16 bytes
 * Size limit L: 65535 with REGK_DNS_TCP, else clamp(requester's OPT size, 512, udp_payload) with OPT and 512 without.
 * Header, question and OPT always; then the longest prefix of the answers that fits in L; only if every answer fit,
 * the longest prefix of the additionals that fits and whose owner pointer is below 0x4000 (a pointer's 14 bits).
 * tc[i] (and the header's TC) is 1 exactly when an answer was left out.
 * launches counts the once-per-resolve preparation (two kernels) on the first call after a resolve only; kernel_ms
 * spans every pass of the call but the host's reads.
 * PARITY UNPINNED (Binder is absent): its rcode for empty non-terminals and names outside its zones; AA and the
 * header bits; answer order and shuffling; its truncation policy; case handling; the form of error responses.  The
 * wire format is RFC 1035, 2782 and 6891.
 * ---- with REGK_DNS_PTR: reverse lookups.  Rules 1-8 are unchanged; rule 9 gains a third kind of owner:
 *   reverse name  exactly six labels o4.o3.o2.o1.in-addr.arpa: the last two equal "in-addr" and "arpa"
 *                 case-insensitively, each octet label 1-3 ASCII digits of value <= 255 without a leading zero ("0"
 *                 is one, "00", "01" and "256" are not); its address is o1.o2.o3.o4.  Any other name, a partial one
 *                 such as 3.2.1.in-addr.arpa included, is not a reverse name.
 *   targets(a)    every snapshot node c with a REGK_Q_HOST_A query whose addr(c) is a, in ascending node order (so
 *                 ops_host and rr_host records, and nodes that are not class OK, are never targets)
 *   A reverse name owns PTR when its address has a target; A and SRV ownership are as above.  QTYPE PTR (12) on a
 *   PTR owner: ANSWER with one PTR RR per target; any other QTYPE on a name that owns A, SRV or PTR: NODATA;
 *   otherwise NXDOMAIN.  node[i] of a PTR answer is its smallest target.
 *   PTR    owner 0xC00C, TYPE 12, CLASS IN, TTL a_ttl(c), RDLENGTH L + 2, name(c) uncompressed (RFC 1035 3.3.12):
 *          14 + L bytes for a name of L text bytes; targets in order
 *   Size limit as above: the longest prefix of the PTR RRs that fits, no additionals; tc is 1 exactly when a PTR RR
 *   was left out.
 *   The reverse index is built once per resolve, on the first REGK_DNS_PTR call after it (launches counts it there:
 *   two compaction kernels, then, when there is a host node, the radix sort as one and two prefix kernels); a call without the flag neither builds nor
 *   drops it and launches exactly the kernels it launched before the flag existed.
 * PARITY UNPINNED (Binder is absent): whether Binder answers PTR at all, its owner set and their order, the TTL, and
 * its rcode for partial reverse names.  The wire format is RFC 1035 3.3.12 and 3.5.
 */
#define REGK_DNS_TCP (1u << 8)      /* regk_dns_opts.flags: a 65535-byte limit (no TCP length prefix is written) */
#define REGK_DNS_PTR (1u << 11)     /* regk_dns_opts.flags: answer PTR for in-addr.arpa names (below) */

typedef struct regk_dns_in {
    const uint8_t  *msgs;           /* k query messages, back to back */
    const uint64_t *off;            /* [k + 1], monotone; message i = msgs[off[i], off[i+1]) */
    uint64_t k, total;              /* total = off[k] (required for device input) */
    uint32_t flags;                 /* REGK_IN_DEVICE */
    uint32_t reserved;              /* 0 */
} regk_dns_in;

typedef struct regk_dns_opts {
    uint32_t flags;                 /* REGK_OUT_DEVICE | REGK_DNS_TCP | REGK_DNS_PTR */
    uint32_t udp_payload;           /* the server's EDNS0 UDP size, 512..65535 (e.g. 1232) */
} regk_dns_opts;

#define REGK_DNS_ANSWER   0u
#define REGK_DNS_NODATA   1u
#define REGK_DNS_NXDOMAIN 2u
#define REGK_DNS_FORMERR  3u
#define REGK_DNS_NOTIMP   4u
#define REGK_DNS_REFUSED  5u
#define REGK_DNS_BADVERS  6u
#define REGK_DNS_DROPPED  7u

typedef struct regk_dns_out {
    uint64_t k, resp_total;
    uint64_t n_status[8];           /* per REGK_DNS_* */
    uint64_t n_truncated;
    uint32_t flags, launches;       /* REGK_OUT_DEVICE */
    const uint64_t *resp_off;       /* [k + 1]; a dropped message has an empty range */
    const uint8_t  *resp;           /* [resp_total] */
    const uint8_t  *status;         /* [k] REGK_DNS_* */
    const uint8_t  *tc;             /* [k] 1 when answers were dropped to fit */
    const uint64_t *node;           /* [k] snapshot node whose records answered, ~0 if none */
    float kernel_ms;
} regk_dns_out;

int         regk_dns_answer(regk_ctx *ctx, const regk_dns_in *in, const regk_dns_opts *opts, regk_dns_out *out);

/*
 * ---- walk a registry subtree: getData and getChildren level by level, into the snapshot regk_resolve answers from
 * (Binder's access pattern, README.md:502-536: fetch the node, list its children, fetch every child) -----------------
 * The walk lives on the context, apart from every batch: finishing a batch does not touch it, and no walk call touches
 * another call's results (regk_read_replies, regk_read_children, regk_resolve, ... stay valid across walk calls).
 * regk_walk_start: the roots (host memory; root i = roots[root_off[i], root_off[i+1]), root_off monotone) are level 0's
 *   frontier, in the order given; any earlier walk is dropped (a refused start leaves it as it was).  REGK_ERR_INVALID_ARG,
 *   naming the smallest bad root:
 *   flags != 0; n_roots == 0; a root ZooKeeper rejects (regk_mkdirp_dirs' INVALID rule, or empty); "/" (its listing would give
 *   "//name", and /zookeeper is not registry data); a root equal to an earlier root; a root that another root is a
 *   proper ancestor of.
 * regk_walk_requests: the current frontier of f nodes as one buffer of 2 f frames - frame i < f is GetDataRequest{path
 *   i, watch = false} = len | xid_base + i | 4 | P | path | 0, frame f + i is GetChildrenRequest{path i, watch = false},
 *   the same layout with op word 8 and xid xid_base + f + i (xids wrap).  The replies can so be read as a getData
 *   section followed, at its end, by a getChildren section.  Framing again (e.g. with a new xid base after a reconnect)
 *   is allowed; the last framing counts.  REGK_ERR_STATE: no walk, or a complete walk (an empty frontier).
 *   REGK_ERR_INVALID_ARG: [xid_base, xid_base + 2 f) covers -1 or -2; f >= 2^30.  flags: REGK_OUT_DEVICE returns
 *   device pointers, else pinned host arrays; valid until the next regk_walk_requests or regk_walk_start.
 * regk_read_walk: bytes[0, len) = what the caller read after sending that framing: the f getData replies, then the f
 *   getChildren replies (host memory, or device memory with REGK_IN_DEVICE, 16-byte aligned).  Notifications (xid -1)
 *   and pings (xid -2) before the last reply are skipped and counted; the stream may go on past the last reply.
 *     found node   frontier node i becomes the next snapshot node iff its getData reply has err 0: its path, the
 *                  reply's data (D = -1 reads as empty), Stat.version and Stat.ephemeralOwner
 *     order        breadth first: level by level, frontier order within a level; level_off holds the boundaries
 *     next level   for each node whose getChildren reply has err 0 (whether or not its getData found it: the two reads
 *                  are separate, and a race between them is not an error), its children in the reply's order, as
 *                  path + '/' + name
 *     errors       NONODE (-101) on either read means the node is gone; any other code is counted in n_error /
 *                  n_list_error: do not trust a snapshot built while either count is nonzero
 *     duplicates   two equal names in one listing are not looked for (a server cannot hold them); regk_resolve would
 *                  refuse the duplicate path, naming the later node
 *   Refusals (REGK_ERR_INVALID_ARG; the message names the byte position and the expected xid): exactly regk_read_replies'
 *   refusals on the getData section and regk_read_children's on the getChildren section, which starts at the getData
 *   section's consumed.  A refused read changes nothing: the frontier, the framing and the snapshot stay as they were,
 *   so the stream can be fixed and read again.  REGK_ERR_STATE: no framing of the current frontier.
 *   The snapshot, version and ephemeral_owner are ALWAYS device arrays, in the layout regk_reconcile takes; level_off is
 *   a host array.  REGK_OUT_DEVICE is accepted and changes nothing.  They stay valid until the next regk_read_walk or
 *   regk_walk_start: a read appends and may reallocate.  A regk_resolve given an earlier walk snapshot must therefore
 *   be redone before regk_dns_answer is used again: a device snapshot passed to that resolve must stay allocated and
 *   unchanged until the last regk_dns_answer on it.  regk_walk_resolve (below) resolves the walk's own snapshot, and
 *   regk_dns_answer refuses to answer from it once the snapshot has changed.
 * PARITY UNPINNED: the layouts are restated from zookeeper.jute and tested against an independent restatement, not
 * against a server.  A directory whose listing exceeds the server's jute.maxbuffer cannot be listed by any client, and
 * this call does not handle it.
 *
 * ---- a watched walk: keep the snapshot current with ZooKeeper watches, as Binder keeps its cache ---------------------
 * regk_walk_requests(..., flags | REGK_ZK_WATCH, ...) writes the trailing watch byte of every frame of both sections as
 *   1; nothing else changes, and without the flag every frame is what it was.  A walk is WATCHED while every level it
 *   has read was framed with the flag (the last framing before each read counts); the two calls below refuse an
 *   unwatched walk with REGK_ERR_STATE.  regk_walk_start drops the marks, the table and the refresh state.
 * Each snapshot node carries two marks: PENDING (re-read it) and REMOVED (drop it).  n_pending counts the nodes that are
 *   pending and not removed, n_removed the removed ones.
 * regk_walk_events: the notifications in bytes[start, len), by exactly regk_read_events' frame rules (opts the same;
 *   notifications, pings, replies in [xid_base, xid_base + n_xids) skipped and counted, a trailing partial frame,
 *   the same refusals, nothing marked on a refusal).  Each event's path is looked up byte for byte among the snapshot's
 *   nodes not marked REMOVED, as the call found them (an event never sees another event of the same call):
 *     NodeDataChanged (3), NodeChildrenChanged (4)   node j becomes PENDING
 *     NodeDeleted (2)                                 j is marked REMOVED (and leaves the pending set); the node at
 *                                                     dirname(path), if it is a node not marked REMOVED, becomes PENDING
 *     any other type, or no such node                 unmatched (node UINT64_MAX); types -1 and 5 .. 7 also count in
 *                                                     n_other
 *   REMOVED wins over PENDING whatever the events' order.  pos, type, state, zxid, node per event are pinned host
 *   arrays, or device arrays with REGK_OUT_DEVICE, valid until the next call.  The path table is brought up to date on the first call
 *   after the snapshot changed: the nodes a level appended are inserted, and after a rebuild (which renumbers the
 *   nodes) or once the table would be over half full it is built anew.  table_nodes / table_ms report the nodes
 *   inserted and that time (0 when the table was current), kernel_ms the rest.
 * regk_walk_refresh (flags 0): on a watched walk with an empty frontier (else REGK_ERR_STATE), (1) drops every REMOVED
 *   node, the survivors keeping their order, data, version, owner and marks; (2) makes the PENDING nodes, ascending, the
 *   frontier of a REFRESH LEVEL and clears the marks; (3) reports n_removed, n_kept, n_frontier, and out->walk: the
 *   walk as it now stands (level 0, level_off = {n_kept}).  No pending node: the walk stays complete.
 * A refresh level is framed by regk_walk_requests as any level (getData and getChildren per node), and regk_read_walk
 *   reads it with these differences:
 *     getData err 0      the node's data, version and owner are replaced in place
 *     getData NONODE     the node is REMOVED; any other err keeps it unchanged (n_error)
 *     getChildren err 0  only the listed children whose path is not a node of the snapshot after this read's
 *                        removals become the next frontier (frontier order, then listing order)
 *     the snapshot       rebuilt once, without every REMOVED node; node ids may change, marks move with their nodes
 *     level_off          {m}: level 0 is the nodes kept from before the refresh, and `level` counts the levels
 *                        appended since (a walk that is never refreshed reports what it always did)
 *   The plain levels after a refresh append as before, but drop every listed child whose path is a node of the snapshot
 *   (REMOVED or not), so the snapshot never holds one path twice and regk_resolve accepts it.
 * ORDERING RULE: every byte the session delivers goes through regk_walk_events exactly once, and bytes that also hold
 *   replies to a walk framing go through regk_read_walk first.  A watch exists only after its read was processed, so a
 *   notification always follows the reply that armed it, and reading replies first maps every event to a present node.
 * WHY NodeDeleted MAKES THE PARENT PENDING: a refresh reads its replies before the events of the same stream.  If node p
 *   is deleted and recreated and its parent g (its child watch already spent) is re-listed after both, g's listing shows
 *   p while the old p is still present, so the new p reads as known; p's NodeDeleted then removes it, and g's child
 *   watch will not fire again.  Making g pending re-lists g once p is gone, so the new p is walked.  A deleted ROOT has
 *   no watched parent: it stays gone until a new walk.
 * CONVERGENCE: once the tree stops changing and every byte has been fed, refreshing until nothing is pending or removed
 *   leaves a snapshot equal, as a set of (path, data, version, owner), to a fresh walk of the same roots (deleted roots
 *   aside); node order differs.  Resolve it with regk_walk_resolve (below), which formats only what changed.  After a
 *   reconnect, carry the walk over with regk_walk_setwatches below; after a session expiry, start a new watched walk.
 * PARITY UNPINNED: restated from zookeeper.jute (WatcherEvent) and the server's watch rules (one-shot, per session; a
 *   getData on a missing node arms nothing; a watch still armed is not duplicated), not tested against a server.
 */
typedef struct regk_walk {
    uint64_t level;                 /* levels read so far */
    uint64_t m;                     /* snapshot nodes so far */
    uint64_t n_frontier;            /* nodes of the next level; 0: the walk is complete */
    uint64_t n_found, n_missing, n_error;               /* this level's getData replies: err 0 / NONODE / other */
    uint64_t n_listed, n_list_missing, n_list_error;    /* this level's getChildren replies, same split */
    uint64_t n_children;            /* listing entries this level read (= the next level's size) */
    uint64_t n_skipped;             /* notifications and pings met before the last reply */
    uint64_t consumed;              /* stream bytes up to the end of the last reply */
    uint32_t flags, launches;
    const uint64_t *level_off;      /* [level + 1], host: level l's nodes are [level_off[l], level_off[l+1]) */
    regk_decode_in  snapshot;       /* ALWAYS device (REGK_IN_DEVICE), aligned as regk_reconcile requires */
    const int32_t  *version;        /* [m] device: Stat.version */
    const int64_t  *ephemeral_owner;/* [m] device: Stat.ephemeralOwner */
    float kernel_ms;
} regk_walk;

int         regk_walk_start(regk_ctx *ctx, const uint8_t *roots, const uint64_t *root_off, uint64_t n_roots, uint32_t flags);
int         regk_walk_requests(regk_ctx *ctx, int32_t xid_base, uint32_t flags, regk_frames *out);
int         regk_read_walk(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint32_t flags, regk_walk *out);

typedef struct regk_walk_events_out {
    uint64_t n_events, n_pings, n_replies;
    uint64_t n_unmatched, n_other;
    uint64_t consumed;              /* end of the last complete frame (start when none) */
    uint64_t n_pending, n_removed;  /* after the call */
    uint64_t table_nodes;           /* nodes this call inserted into the path table; 0: it was current */
    uint32_t partial;               /* 1: a frame starts at consumed and the stream ends inside it */
    uint32_t flags, launches;       /* REGK_OUT_DEVICE */
    uint32_t reserved;
    const uint64_t *pos;            /* [n_events] the frame's first byte */
    const int32_t  *type;           /* WatcherEvent.type */
    const int32_t  *state;          /* WatcherEvent.state */
    const int64_t  *zxid;           /* ReplyHeader.zxid */
    const uint64_t *node;           /* the snapshot node, or UINT64_MAX */
    float kernel_ms;                /* the events, without the table build */
    float table_ms;                 /* the table build */
} regk_walk_events_out;

typedef struct regk_walk_refresh_out {
    uint64_t n_removed, n_kept, n_frontier;
    uint32_t flags, launches;
    regk_walk walk;                 /* the walk after the refresh: level 0, level_off {n_kept}, the compacted snapshot */
    float kernel_ms;
} regk_walk_refresh_out;

int         regk_walk_events(regk_ctx *ctx, const uint8_t *bytes, uint64_t len, uint64_t start, const regk_events_opts *opts,
                             regk_walk_events_out *out);
int         regk_walk_refresh(regk_ctx *ctx, uint32_t flags, regk_walk_refresh_out *out);

/*
 * ---- a watched walk across a reconnect: ZooKeeper drops a connection's watches with the connection, though the
 * session survives.  regk_walk_setwatches frames SetWatches (op 101) for the watches the walk's session holds, so the
 * server re-arms them on the new connection or fires what the walk missed, and re-pends every other node -------------
 * ARMED: each snapshot node carries one more bit, set when the last read of the node (the plain level that appended it,
 *   or a refresh level that re-read it) was framed with REGK_ZK_WATCH and both its getData and its getChildren reply had
 *   err 0.  Any other outcome clears it: an unwatched framing, a refresh-level getData err other than NONODE (which
 *   arms nothing), a getChildren err (no child watch).  The bit moves with its node through a rebuild, and
 *   regk_walk_start clears everything.  This bookkeeping, and the mark's below, is not counted in any call's
 *   `launches`.
 * The walk's zxid high-water mark is the largest ReplyHeader.zxid of every reply frame a successful regk_read_walk read
 *   (both sections' frame chains, not the listing entries) and of every reply and SetWatches reply a successful
 *   regk_walk_events walked; never a notification or a ping.  A refused call does not move it, regk_walk_start resets it
 *   to 0, and it is the walk's own, apart from the heartbeat's: an overestimate loses events, and only the bytes this
 *   walk read vouch for it.  It is safe as relativeZxid for the reason the heartbeat's is: a reply with zxid R leaves the
 *   server after every notification of a change at or below R, and TCP keeps that order.  The ORDERING RULE feeds every
 *   delivered byte through regk_walk_events, so a change the walk missed was notified after the last reply it read,
 *   and its zxid is above the mark: the server fires it again.  An underestimate only fires spurious events.
 *
 * regk_walk_setwatches (opts as regk_setwatches_requests takes them): on a watched walk (else REGK_ERR_STATE), complete
 *   or with a level in flight.  Call it when the connection drops, before reconnecting; relative_zxid is also the
 *   ConnectRequest's lastZxidSeen.
 *     LISTED     every node that is ARMED and neither PENDING, REMOVED nor a node of the refresh frontier (a refresh
 *                level framed or about to be), ascending, into D (data watches); the same nodes in the same order
 *                into C (child watches); E is empty.
 *     RE-PENDED  every other node that is neither PENDING, REMOVED nor of the refresh frontier becomes PENDING
 *                (n_repend), so the next refresh re-reads and re-arms it.
 *     LEFT ALONE pending and removed nodes, and the frontier: n_frontier (0: none) is the level to frame again after the
 *                reconnect with regk_walk_requests, whose reads arm those nodes.
 *   Frames: exactly regk_setwatches_requests' layout and split, with Lmax = 4 + the snapshot's longest path; max_frame's
 *   default, bounds and refusal (naming the minimum) are the same.  Pinned host arrays, or device arrays with
 *   REGK_OUT_DEVICE, valid until the next call.  A refused call changes nothing, and every buffer is reserved before any
 *   node is re-pended.  After a successful call regk_walk_events also accepts a SetWatches reply (xid -8, len 16,
 *   err 0: skipped, counted in n_replies, its zxid entering the mark); a -8 frame with a body or an err is refused.
 *   Before any such call -8 is refused as any negative xid; regk_walk_start closes the gate.  regk_read_walk is unchanged.
 * RECONNECT PROTOCOL:
 *   1. Feed every delivered byte through regk_walk_events as usual.  The bytes of a level whose replies were cut off may
 *      be fed with that level's reply range, or discarded: an event fed is a real change, and an event discarded was
 *      notified after every reply the walk read, so its zxid is above the mark and SetWatches fires it again.
 *   2. Call regk_walk_setwatches, and reconnect with lastZxidSeen = relative_zxid.
 *   3. Send the SetWatches frames.
 *   4. Feed the stream through regk_walk_events until every SetWatches reply has been seen (one per frame).  The
 *      notifications the server fires from DataTree.setWatches arrive before each reply and mark the nodes that changed.
 *      A deleted node, listed in D and in C, fires NodeDeleted twice; REMOVED is idempotent.
 *   5. If n_frontier > 0, frame that level again (regk_walk_requests, a fresh xid base) and read it as usual.
 *   6. Refresh as usual.
 * CONVERGENCE: a walk carried over this way converges as a watched walk does: once the tree stops changing, refreshing
 *   until nothing is pending or removed leaves the set of a fresh walk of the same roots, deleted roots aside; then
 *   regk_walk_resolve brings the answers up to date, re-read nodes whose data did not change keeping their text.  A
 *   session expiry still means a new walk.
 * PARITY UNPINNED: the server's re-arming is restated from ZooKeeper 3.4's DataTree.setWatches, not tested against a
 *   server.
 */
typedef struct regk_walk_setwatches_out {
    uint64_t n_listed;              /* snapshot nodes listed (each once in D and once in C) */
    uint64_t n_repend;              /* nodes this call made PENDING */
    uint64_t n_pending, n_removed;  /* after the call, as regk_walk_events reports them */
    uint64_t n_frontier;            /* the level in flight, to be framed again after the reconnect; 0: none */
    int64_t  relative_zxid;
    regk_frames frames;
} regk_walk_setwatches_out;

int         regk_walk_setwatches(regk_ctx *ctx, const regk_setwatches_opts *opts, regk_walk_setwatches_out *out);

/*
 * ---- a walk's answers kept current: re-resolve the walk's snapshot as it stands, reusing the last call's text for
 * every answer whose inputs did not change -----------------------------------------------------------------------------
 * regk_walk_resolve: REGK_ERR_STATE when there is no walk; batches in flight are refused as regk_resolve refuses them.
 *   A walk in any phase is accepted (a level in flight, REMOVED nodes not yet refreshed, complete): what is resolved is
 *   the walk's snapshot as it stands, which is what regk_resolve(ctx, &walk.snapshot, opts, ...) sees.
 * RESULT: out->answers has every count (m, n_queries, n_answers, n_additional, n_unresolved, text_total) and every
 *   array (q_kind, q_node, sec_off, text, node_cls, unresolved) byte-identical to what that regk_resolve would return;
 *   launches and kernel_ms are this call's own.  opts is validated as regk_resolve validates it (the same refusals,
 *   and the same refusal of a duplicate path naming the later node), the message naming this call.  Pinned host arrays,
 *   or device arrays with REGK_OUT_DEVICE, valid until the next regk_walk_resolve, regk_resolve or regk_walk_start.
 * regk_dns_answer then answers from this call as it answers after regk_resolve, byte for byte.  Once the walk's
 *   snapshot has changed since the call (a regk_read_walk that appended or rebuilt, a regk_walk_refresh that rebuilt,
 *   a regk_walk_start), regk_dns_answer returns REGK_ERR_STATE: resolve again.  After a plain regk_resolve it behaves as
 *   it always did.
 * IDENTITY: each walk snapshot node has an identity (its index at the last successful regk_walk_resolve) or none.
 *   After a successful call every node has one.  A node a plain level appends has none.  A refresh-level getData with
 *   err 0 takes a node's identity only when the new data bytes differ from its old ones (length or any byte); version
 *   and owner enter no answer, so a re-read of unchanged data (e.g. of a node regk_walk_setwatches re-pended) keeps it.
 *   The identity moves with its node through every rebuild, a node dropped as REMOVED takes it along, and
 *   regk_walk_start clears everything, the kept text included.  This bookkeeping is not counted in any walk call's
 *   launches or kernel_ms, and no walk call's outputs change.
 * REUSE: full = 1 when there was no successful regk_walk_resolve since the last regk_walk_start, or its
 *   default_host_ttl / default_srv_ttl or REGK_RESOLVE_ANY_FORM differ from this call's: n_fresh = m, copied_bytes = 0, every line formatted.
 *   Otherwise a HOST_A section is copied from the last call's text when its node has an identity, and a service child's
 *   A line, SRV lines and additional line when the child and its service both have one; everything else is formatted.
 *   This is exact: a node's class, roles and TTL depend only on its own path, data and opts; whether a node is a child
 *   of a service, and the child's lines, depend only on the two of them; a node's path never changes.  So a copied run
 *   holds the bytes regk_resolve would write.
 * A refused or failed call keeps the last successful call's text and every identity (and, as regk_resolve, leaves no
 *   answers for regk_dns_answer).  A plain regk_resolve in between does not break reuse: the kept text is this call's.
 * The option "walk_resolve_segments" (regk_get_option) reports the last successful call's segments: the runs its text
 *   was assembled from (0 when full).
 */
typedef struct regk_walk_answers {
    regk_answers answers;           /* exactly regk_resolve's outputs for the walk's snapshot as it stands */
    uint64_t n_fresh;               /* snapshot nodes without an identity at the last regk_walk_resolve (all m when full) */
    uint64_t copied_bytes;          /* text bytes taken from the last regk_walk_resolve's text */
    uint64_t formatted_bytes;       /* text_total - copied_bytes */
    uint32_t full;                  /* 1: nothing to reuse, every line formatted */
    uint32_t reserved;
} regk_walk_answers;

int         regk_walk_resolve(regk_ctx *ctx, const regk_resolve_opts *opts, regk_walk_answers *out);

/* Tuning knobs (kernel variant selection for A/B measurement); see DESIGN.md. */
int         regk_set_option(regk_ctx *ctx, const char *name, int64_t value);
int64_t     regk_get_option(const regk_ctx *ctx, const char *name);

#ifdef __cplusplus
}
#endif
#endif /* REGK_H */
