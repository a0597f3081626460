/*
 * dns_emul.cpp — TEST INFRASTRUCTURE: the per-message rules of regk_dns.cuh (dns_parse, dns_path, dns_limit) and the
 * truncation arithmetic (dns_fit, dns_resp_len) on the CPU.  Built as a standalone program with
 * -fsanitize=address,undefined by tests/test_dns_cpu.py: every message and every array is allocated with exactly its
 * length, so a read past its end stops the program.  Not part of the product library.
 *
 * stdin, one command per line:
 *   P <message hex or ->                   -> <status> <qend> <name> <labels> <qtype> <qclass> <opt> <do> <req> <plain>
 *                                             <path hex or ->  (the path when the name parsed and has labels)
 *   F <kind> <L> <qend> <opt> <n> <np_0> <len_0> ... <np_n-1> <len_n-1>
 *                                          -> <nans> <nadd> <ans_bytes> <tc> <response bytes>
 *      (a service's children with np SRV RRs of 20 + len bytes each; host A: n = 0)
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../registrar_b200/csrc/regk_dns.cuh"

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

int main()
{
    static char line[1 << 20];
    while (fgets(line, sizeof line, stdin)) {
        const char *cmd = strtok(line, " \n");
        if (!cmd)
            continue;
        if (cmd[0] == 'P') {
            uint32_t n = 0;
            uint8_t *m = unhex(strtok(nullptr, " \n"), &n);
            const DnsMsg r = dns_parse(m, n);
            printf("%u %u %u %u %u %u %u %u %u %u ", r.status, r.qend, r.name, r.labels, r.qtype, r.qclass, r.opt, r.dobit,
                r.req_size, r.plain);
            if (r.qend && r.labels) {
                const uint32_t pl = r.name - 1u;
                uint8_t *path = (uint8_t *)malloc(pl);
                if (dns_path(m + 12, r.name, path) != pl)
                    return 3;
                for (uint32_t k = 0; k < pl; k++)
                    printf("%02x", path[k]);
                free(path);
            } else {
                printf("-");
            }
            printf("\n");
            free(m);
        } else {
            const uint32_t kind = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            const uint32_t L = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            const uint32_t qend = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            const uint32_t opt = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            const uint32_t n = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            unsigned long long *S = (unsigned long long *)malloc((n + 1) * 8), *N = (unsigned long long *)malloc((n + 1) * 8),
                               *A = (unsigned long long *)malloc((n + 1) * 8);
            S[0] = N[0] = A[0] = 0;
            for (uint32_t c = 0; c < n; c++) {
                const unsigned long long np = strtoull(strtok(nullptr, " \n"), nullptr, 10);
                const unsigned long long len = strtoull(strtok(nullptr, " \n"), nullptr, 10);
                S[c + 1] = S[c] + np * (20u + len);
                N[c + 1] = N[c] + np;
                A[c + 1] = A[c] + (np ? 1u : 0u);
            }
            const DnsFit f = dns_fit(kind, 0, n, S, N, A, L, qend + (opt ? DNS_OPT_RR : 0u), qend);
            printf("%u %u %u %u %u\n", f.nans, f.nadd, f.ans_bytes, f.tc, dns_resp_len(DNS_ANSWER, qend, opt, f.ans_bytes, f.nadd));
            free(S);
            free(N);
            free(A);
        }
    }
    return 0;
}
