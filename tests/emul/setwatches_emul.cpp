/*
 * setwatches_emul.cpp — TEST INFRASTRUCTURE: the SetWatches helpers of regk_setwatches.cuh on the CPU: the reader's
 * test with SetWatches replies accepted (ev_sw_head), its register formulation (ev_sw_mask16), and the closed-form
 * frame and entry positions (sw_frame_off, sw_entry_pos).  Built as a standalone program with
 * -fsanitize=address,undefined by tests/test_setwatches_cpu.py: the stream is allocated with exactly its length, so a
 * read past its end stops the program.  Not part of the product library.
 *
 * stdin, one command per line:
 *   S <hex or ->            the stream
 *   X <xid_base> <n>        the reply range
 *   P                       ev_sw_head at every position: one code per position
 *   M                       ev_sw_mask16 over every 16-byte block, fed as the candidate kernel feeds it: one 0 / 1
 *                           per position
 *   E <B> <list> <s...>     sw_entry_pos of each prefix s
 *   F <f> <s_first>         sw_frame_off
 * Results on stdout, whitespace separated, one line per command that prints.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../registrar_b200/csrc/regk_setwatches.cuh"

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
    static char line[1 << 20];
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
                printf("%u ", ev_sw_head(s + pos, len - pos, xb, n, &h));
            }
            printf("\n");
        } else if (line[0] == 'M') {
            for (uint64_t at = 0; at < len; at += 16) {
                uint8_t blk[48] = {0};
                memcpy(blk, s + at, len - at < 48 ? len - at : 48);
                uint32_t w[12];
                for (int q = 0; q < 12; q++)
                    w[q] = (uint32_t)blk[4 * q] | (uint32_t)blk[4 * q + 1] << 8 | (uint32_t)blk[4 * q + 2] << 16 |
                           (uint32_t)blk[4 * q + 3] << 24;
                const uint32_t m = ev_sw_mask16(w, len - at, 0u, xb, n);
                for (uint64_t f = 0; f < 16 && at + f < len; f++)
                    printf("%u ", (m >> f) & 1u);
            }
            printf("\n");
        } else if (line[0] == 'E') {
            const uint64_t B = strtoull(strtok(line + 2, " \n"), nullptr, 10);
            const uint32_t list = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            for (char *t = strtok(nullptr, " \n"); t; t = strtok(nullptr, " \n"))
                printf("%llu ", (unsigned long long)sw_entry_pos(strtoull(t, nullptr, 10), B, list));
            printf("\n");
        } else if (line[0] == 'F') {
            const uint64_t f = strtoull(strtok(line + 2, " \n"), nullptr, 10);
            printf("%llu\n", (unsigned long long)sw_frame_off(f, strtoull(strtok(nullptr, " \n"), nullptr, 10)));
        }
        fflush(stdout);
    }
    free(s);
    return 0;
}
