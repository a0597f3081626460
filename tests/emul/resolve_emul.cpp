/*
 * resolve_emul.cpp — TEST INFRASTRUCTURE: the per-node rules of regk_resolve.cuh (rv_classify with its name, IPv4 and
 * ttl checks, the line lengths and the line writers) on the CPU, after regk_decode's per-record logic with
 * host_nodes = 0.  Built as a standalone program with -fsanitize=address,undefined by tests/test_resolve_cpu.py: every
 * input is allocated with exactly its length, so a read past its end stops the program.  Not part of the product
 * library.
 *
 * stdin, one node per line:  <path hex or -> <data hex or -> <default_host_ttl> <default_srv_ttl>
 * stdout, one line per node: <class> <roles> <ttl> <line hex or ->
 *   line: a HOST_A node's A line; a service's SRV line to the child "c.x" at the service's own port (its length checked
 *   against rv_srv_len); otherwise "-".
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../registrar_b200/csrc/regk_resolve.cuh"

using namespace regk;

static uint8_t *unhex(const char *hex, uint32_t *len)
{
    *len = strcmp(hex, "-") ? (uint32_t)(strlen(hex) / 2) : 0u;
    uint8_t *b = (uint8_t *)malloc(*len ? *len : 1);
    for (uint32_t i = 0; i < *len; i++) {
        unsigned v;
        sscanf(hex + 2 * i, "%2x", &v);
        b[i] = (uint8_t)v;
    }
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
        uint32_t pn = 0, jn = 0;
        uint8_t *path = unhex(ph, &pn), *json = unhex(jh, &jn);
        uint8_t *dom = (uint8_t *)malloc(pn ? pn : 1);
        uint32_t *ports = (uint32_t *)malloc((jn / 2 + 1) * sizeof(uint32_t));
        Decoded d;
        d.flags = decode_path(path, pn, false, dom, d);
        d.flags |= decode_payload<true>(json, jn, d, ports);
        const RvNode r = rv_classify(d, json, jn, dom, ports, dh, ds);
        printf("%u %u %d ", r.cls, r.roles, r.ttl);
        std::vector<uint8_t> out;
        if (r.roles & RV_ROLE_HOST_A) {
            out.resize(rv_a_len(d.dom_len, r.ttl, d.addr_len));
            const uint8_t *e = rv_put_a(out.data(), dom, d.dom_len, r.ttl, json + d.addr_pos, d.addr_len);
            if ((uint64_t)(e - out.data()) != out.size())
                return 3;
        } else if (r.roles & RV_ROLE_SERVICE) {
            static const uint8_t child[] = {'c', '.', 'x'};
            out.resize(rv_srv_len(d.type_len, d.addr_len, d.dom_len, r.ttl, ports[0], 3));
            const uint8_t *e = rv_put_srv(out.data(), json + d.type_pos, d.type_len, json + d.addr_pos, d.addr_len, dom, d.dom_len,
                r.ttl, ports[0], child, 3);
            if ((uint64_t)(e - out.data()) != out.size())
                return 3;
        }
        put_hex(out.data(), out.size());
        printf("\n");
        free(path);
        free(json);
        free(dom);
        free(ports);
    }
    return 0;
}
