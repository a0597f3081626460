/*
 * resolve_any_emul.cpp — TEST INFRASTRUCTURE: REGK_RESOLVE_ANY_FORM's per-node path on the CPU: regk_decode's
 * per-record logic (host_nodes = 0), the candidate test and the general reader of regk_resolve_any.cuh, then
 * rv_classify<true>.  Built as a standalone program with -fsanitize=address,undefined by tests/test_resolve_any_cpu.py:
 * every payload is allocated with exactly its length, so the GUARD reader is checked flush against the end of its
 * buffer; the word-load reader runs on a copy with 16 bytes of slack and must agree.  Not part of the product library.
 *
 * stdin, one node per line:  <path hex or -> <data hex or -> <default_host_ttl> <default_srv_ttl>
 * stdout, one line per node: <class> <roles> <ttl> <read> <kind> <type hex or -> <addr hex or -> <nports> <ports,...>
 *   read: 1 when the general reader read the node; kind/type/addr/ports: the record classify saw ('h' host, 's'
 *   service; '-' with class NOT_RECORD or EMPTY); nports -1 for a host record without ports.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../registrar_b200/csrc/regk_resolve_any.cuh"

using namespace regk;

static uint8_t *unhex(const char *hex, uint32_t *len, uint32_t slack)
{
    *len = strcmp(hex, "-") ? (uint32_t)(strlen(hex) / 2) : 0u;
    uint8_t *b = (uint8_t *)malloc(*len + slack ? *len + slack : 1);
    for (uint32_t i = 0; i < *len; i++) {
        unsigned v;
        sscanf(hex + 2 * i, "%2x", &v);
        b[i] = (uint8_t)v;
    }
    for (uint32_t i = 0; i < slack; i++)
        b[*len + i] = (uint8_t)(0x22 + i);              /* quotes and the like behind the end */
    return b;
}

static void put_hex(const uint8_t *b, uint64_t n)
{
    if (!n)
        printf("-");
    for (uint64_t i = 0; i < n; i++)
        printf("%02x", b[i]);
}

int main()
{
    static char line[1 << 20];
    while (fgets(line, sizeof line, stdin)) {
        const char *ph = strtok(line, " \n"), *jh = strtok(nullptr, " \n");
        const int32_t dh = (int32_t)strtol(strtok(nullptr, " \n"), nullptr, 10);
        const int32_t ds = (int32_t)strtol(strtok(nullptr, " \n"), nullptr, 10);
        uint32_t pn = 0, jn = 0, jn2 = 0;
        uint8_t *path = unhex(ph, &pn, 0), *json = unhex(jh, &jn, 0), *json2 = unhex(jh, &jn2, 16);
        uint8_t *dom = (uint8_t *)malloc(pn ? pn : 1);
        const size_t np = jn / 2 + 1;
        uint32_t *ports = (uint32_t *)malloc(np * sizeof(uint32_t)), *ports2 = (uint32_t *)malloc(np * sizeof(uint32_t));
        Decoded d;
        memset(&d, 0, sizeof d);
        d.ttl = INT32_MIN;
        d.nports = 0xFFFFFFFFu;
        d.flags = decode_path(path, pn, false, dom, d);
        d.flags |= decode_payload<true>(json, jn, d, ports);
        memcpy(ports2, ports, np * sizeof(uint32_t));
        Decoded d2 = d;
        bool read = false;
        if (any_candidate(d, jn)) {
            read = read_any<true>(json, jn, d, ports);
            const bool read2 = read_any<false>(json2, jn2, d2, ports2);
            if (read != read2 || memcmp(&d, &d2, sizeof d) != 0)
                return 4;                                   /* the two cursors disagree */
            if (read && d.nports != 0xFFFFFFFFu && memcmp(ports, ports2, d.nports * sizeof(uint32_t)) != 0)
                return 4;
        }
        const RvNode r = rv_classify<true>(d, json, jn, dom, ports, dh, ds);
        printf("%u %u %d %d ", r.cls, r.roles, r.ttl, read ? 1 : 0);
        if (r.cls >= RV_BAD_NAME || r.cls == RV_OK) {
            const bool svc = (d.flags & DEC_SERVICE_RECORD) != 0;
            printf("%c ", svc ? 's' : 'h');
            put_hex(json + d.type_pos, d.type_len);
            printf(" ");
            put_hex(json + d.addr_pos, d.addr_len);
            const uint32_t n = d.nports;
            printf(" %d ", n == 0xFFFFFFFFu ? -1 : (int)n);
            if (n == 0xFFFFFFFFu || n == 0)
                printf("-");
            for (uint32_t k = 0; n != 0xFFFFFFFFu && k < n; k++)
                printf(k ? ",%u" : "%u", ports[k]);
        } else {
            printf("- - - 0 -");
        }
        printf("\n");
        free(path);
        free(json);
        free(json2);
        free(dom);
        free(ports);
        free(ports2);
    }
    return 0;
}
