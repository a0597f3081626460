/*
 * events_emul.cpp — TEST INFRASTRUCTURE: the per-frame test of regk_events.cuh (ev_head) and its register formulation
 * (ev_mask16) on the CPU.  Built as a standalone program with -fsanitize=address,undefined by tests/test_events_cpu.py:
 * the stream is allocated with exactly its length, so a read past its end stops the program.  Not part of the product
 * library.
 *
 * stdin, one command per line:
 *   S <hex or ->            the stream
 *   X <xid_base> <n>        the reply range
 *   P                       ev_head at every position: one code per position
 *   M <first>               ev_mask16 over every 16-byte block, fed as the candidate kernel feeds it (the block and the
 *                           two after it as little-endian words, zero past the stream's end): one 0 / 1 per position
 *   R <start>               the stream walked front to back with ev_head, as regk_read_events walks it: "0 <consumed>
 *                           <partial> <pings> <replies> <pos type state zxid path-length of every event...>", or
 *                           "<code> <position>"
 * Results on stdout, whitespace separated.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../registrar_b200/csrc/regk_events.cuh"

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
                EvHead h;
                printf("%u ", ev_head(s + pos, len - pos, xb, n, &h));
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
                const uint32_t m = ev_mask16(w, len - at, first > at ? (uint32_t)(first - at > 16 ? 16 : first - at) : 0u, xb, n);
                for (uint64_t f = 0; f < 16 && at + f < len; f++)
                    printf("%u ", (m >> f) & 1u);
            }
            printf("\n");
        } else if (line[0] == 'R') {
            uint64_t pos = strtoull(line + 2, nullptr, 10), pings = 0, replies = 0;
            std::vector<long long> ev;
            uint32_t code = EV_OK;
            bool partial = false;
            while (pos < len) {
                EvHead h;
                code = ev_head(s + pos, len - pos, xb, n, &h);
                if (code == EV_TRUNC) {
                    partial = true;
                    code = EV_OK;
                    break;
                }
                if (code != EV_OK)
                    break;
                if (h.kind == RK_NOTIFY) {
                    const uint8_t *fr = s + pos;
                    ev.push_back((long long)pos);
                    ev.push_back(h.type);
                    ev.push_back((int32_t)be32_at(fr + 24));
                    ev.push_back((long long)((unsigned long long)be32_at(fr + 8) << 32 | be32_at(fr + 12)));
                    ev.push_back(h.plen);
                } else if (h.kind == RK_PING) {
                    pings++;
                } else {
                    replies++;
                }
                pos += 4u + (uint32_t)h.len;
            }
            if (code != EV_OK) {
                printf("%u %llu\n", code, (unsigned long long)pos);
            } else {
                printf("0 %llu %d %llu %llu", (unsigned long long)pos, partial ? 1 : 0, (unsigned long long)pings,
                    (unsigned long long)replies);
                for (long long v : ev)
                    printf(" %lld", v);
                printf("\n");
            }
        }
        fflush(stdout);
    }
    free(s);
    return 0;
}
