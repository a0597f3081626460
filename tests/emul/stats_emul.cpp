/*
 * stats_emul.cpp — TEST INFRASTRUCTURE: the per-frame helpers of regk_stats.cuh (stat_head, stat_check) and the register
 * formulation of the candidate test (stat_mask16) on the CPU.  Built as a standalone program with
 * -fsanitize=address,undefined by tests/test_stats_cpu.py: the stream is allocated with exactly its length, so a read past
 * its end stops the program.  Not part of the product library.
 *
 * stdin, one command per line:
 *   S <hex or ->            the stream
 *   X <xid_base> <n>        the framing
 *   P                       stat_head at every position: one code per position
 *   M <first>               stat_mask16 over every 16-byte block, fed as the candidate kernel feeds it (the block and the
 *                           two after it as little-endian words, zero past the stream's end): one 0 / 1 per position;
 *                           positions below <first> are left out
 *   R <start>               the stream read front to back with stat_check, as regk_read_stats reads it: "0 <consumed>
 *                           <skipped> <err version owner dataLength mzxid of every record...>", or "<code> <position>
 *                           <record>"
 * Results on stdout, whitespace separated.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../registrar_b200/csrc/regk_stats.cuh"

using namespace regk;

static uint8_t *unhex(const char *hex, uint64_t *len)
{
    *len = strcmp(hex, "-") ? strlen(hex) / 2 : 0;
    uint8_t *b = (uint8_t *)malloc(*len ? *len : 1);
    for (uint64_t i = 0; i < *len; i++) {
        unsigned v;
        sscanf(hex + 2 * i, "%2x", &v);
        b[i] = (uint8_t)v;
    }
    return b;
}

static long long be64(const uint8_t *b)
{
    return (long long)((unsigned long long)be32_at(b) << 32 | be32_at(b + 4));
}

int main()
{
    static char line[1 << 22];
    uint8_t *s = nullptr;
    uint64_t len = 0, n = 0;
    int32_t xb = 0;
    while (fgets(line, sizeof line, stdin)) {
        if (line[0] == 'S') {
            free(s);
            s = unhex(strtok(line + 2, " \n"), &len);
        } else if (line[0] == 'X') {
            xb = (int32_t)strtol(strtok(line + 2, " \n"), nullptr, 10);
            n = strtoull(strtok(nullptr, " \n"), nullptr, 10);
        } else if (line[0] == 'P') {
            for (uint64_t pos = 0; pos < len; pos++) {
                StatHead h;
                printf("%u ", stat_head(s + pos, len - pos, xb, n, &h));
            }
            printf("\n");
        } else if (line[0] == 'M') {
            const uint64_t first = strtoull(line + 2, nullptr, 10);
            for (uint64_t at = 0; at < len; at += 16) {
                uint8_t blk[48] = {0};
                memcpy(blk, s + at, len - at < 48 ? len - at : 48);
                uint32_t w[12];
                for (int q = 0; q < 12; q++)
                    w[q] = (uint32_t)blk[4 * q] | (uint32_t)blk[4 * q + 1] << 8 | (uint32_t)blk[4 * q + 2] << 16 |
                           (uint32_t)blk[4 * q + 3] << 24;
                const uint32_t m = stat_mask16(w, len - at, first > at ? (uint32_t)(first - at > 16 ? 16 : first - at) : 0u, xb, n);
                for (uint64_t f = 0; f < 16 && at + f < len; f++)
                    printf("%u ", (m >> f) & 1u);
            }
            printf("\n");
        } else if (line[0] == 'R') {
            uint64_t pos = strtoull(line + 2, nullptr, 10), k = 0, skipped = 0;
            std::vector<long long> rec;
            uint32_t code = ST_OK;
            while (k < n) {
                StatHead h;
                code = stat_check(s + pos, len - pos, xb, n, k, &h);
                if (code != ST_OK)
                    break;
                if (h.kind == RK_REPLY) {
                    const uint8_t *fr = s + pos;
                    const bool found = h.err == 0;
                    rec.push_back(h.err);
                    rec.push_back(found ? (int32_t)be32_at(fr + 52) : 0);
                    rec.push_back(found ? be64(fr + 64) : 0);
                    rec.push_back(found ? (int32_t)be32_at(fr + 72) : 0);
                    rec.push_back(found ? be64(fr + 28) : 0);
                    k++;
                } else {
                    skipped++;
                }
                pos += 4u + (uint32_t)h.len;
            }
            if (code != ST_OK) {
                printf("%u %llu %llu\n", code, (unsigned long long)pos, (unsigned long long)k);
            } else {
                printf("0 %llu %llu", (unsigned long long)pos, (unsigned long long)skipped);
                for (long long v : rec)
                    printf(" %lld", v);
                printf("\n");
            }
        }
        fflush(stdout);
    }
    free(s);
    return 0;
}
