/*
 * replies_emul.cpp — TEST INFRASTRUCTURE: the per-frame helpers of regk_replies.cuh (reply_head, reply_check) on the
 * CPU.  Built as a standalone program with -fsanitize=address,undefined by tests/test_replies_cpu.py: the stream is
 * allocated with exactly its length, so a read past its end stops the program.  Not part of the product library.
 *
 * stdin, one command per line:
 *   S <hex or -> <xid_base> <n>   the stream and the framed requests
 *   P                             reply_head at every position: one code per position
 *   R                             the stream read front to back with reply_check, as regk_read_replies reads it:
 *                                 "0 <consumed> <skipped> <err of every record>", or "<code> <position> <record>"
 * Results on stdout, whitespace separated.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../registrar_b200/csrc/regk_replies.cuh"

using namespace regk;

int main()
{
    static char line[1 << 22];
    uint8_t *s = nullptr;
    uint64_t len = 0, n = 0;
    int32_t xb = 0;
    while (fgets(line, sizeof line, stdin)) {
        if (line[0] == 'S') {
            char *hex = strtok(line + 2, " \n");
            xb = (int32_t)strtol(strtok(nullptr, " \n"), nullptr, 10);
            n = strtoull(strtok(nullptr, " \n"), nullptr, 10);
            free(s);
            len = strcmp(hex, "-") ? strlen(hex) / 2 : 0;
            s = (uint8_t *)malloc(len ? len : 1);
            for (uint64_t i = 0; i < len; i++) {
                unsigned v;
                sscanf(hex + 2 * i, "%2x", &v);
                s[i] = (uint8_t)v;
            }
        } else if (line[0] == 'P') {
            for (uint64_t pos = 0; pos < len; pos++) {
                ReplyHead h;
                printf("%u ", reply_head(s + pos, len - pos, xb, n, &h));
            }
            printf("\n");
        } else if (line[0] == 'R') {
            uint64_t pos = 0, k = 0, skipped = 0;
            std::vector<int32_t> err;
            uint32_t code = RP_OK;
            while (k < n) {
                ReplyHead h;
                code = reply_check(s + pos, len - pos, xb, n, k, &h);
                if (code != RP_OK)
                    break;
                if (h.kind == RK_REPLY) {
                    err.push_back(h.err);
                    k++;
                } else {
                    skipped++;
                }
                pos += 4u + (uint32_t)h.len;
            }
            if (code != RP_OK) {
                printf("%u %llu %llu\n", code, (unsigned long long)pos, (unsigned long long)k);
            } else {
                printf("0 %llu %llu", (unsigned long long)pos, (unsigned long long)skipped);
                for (int32_t e : err)
                    printf(" %d", e);
                printf("\n");
            }
        }
        fflush(stdout);
    }
    free(s);
    return 0;
}
