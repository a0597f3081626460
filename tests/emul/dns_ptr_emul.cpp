/*
 * dns_ptr_emul.cpp — TEST INFRASTRUCTURE: the reverse-name recogniser (dns_reverse) and the PTR truncation cut
 * (dns_fit_ptr) of regk_dns_ptr.cuh on the CPU.  Built as a standalone program with -fsanitize=address,undefined by
 * tests/test_dns_ptr_cpu.py: every message and every array is allocated with exactly its length, so a read past its
 * end stops the program.  Not part of the product library.
 *
 * stdin, one command per line:
 *   R <message hex or ->                   -> <status> <address, or - when not a reverse name>
 *   C <room> <n> <len_0> ... <len_n-1>     -> <nans> <ans_bytes> <tc>   (PTR RRs of 14 + len bytes each)
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../registrar_b200/csrc/regk_dns_ptr.cuh"

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
        if (cmd[0] == 'R') {
            uint32_t n = 0;
            uint8_t *m = unhex(strtok(nullptr, " \n"), &n);
            const DnsMsg r = dns_parse(m, n);
            const uint64_t a = r.status == DNS_ANSWER ? dns_reverse(m + 12, r.labels) : DNS_NOT_REVERSE;
            if (a == DNS_NOT_REVERSE)
                printf("%u -\n", r.status);
            else
                printf("%u %llu\n", r.status, (unsigned long long)a);
            free(m);
        } else {
            const uint32_t room = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            const uint32_t n = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            unsigned long long *B = (unsigned long long *)malloc((n + 1) * 8);
            B[0] = 0;
            for (uint32_t c = 0; c < n; c++)
                B[c + 1] = B[c] + DNS_PTR_RR + strtoull(strtok(nullptr, " \n"), nullptr, 10);
            const DnsFit f = dns_fit_ptr(B, 0, n, room);
            printf("%u %u %u\n", f.nans, f.ans_bytes, f.tc);
            free(B);
        }
    }
    return 0;
}
