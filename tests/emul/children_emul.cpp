/*
 * children_emul.cpp — TEST INFRASTRUCTURE: the per-frame helpers of regk_children.cuh (children_head, children_check,
 * children_entry) on the CPU.  Built as a standalone program with -fsanitize=address,undefined by
 * tests/test_children_cpu.py: the stream is allocated with exactly its length, so a read past its end stops the program.
 * Not part of the product library.
 *
 * stdin, one command per line:
 *   S <hex or -> <xid_base> <d>   the stream and the framed requests
 *   P                             children_head at every position: one code per position
 *   R <start>                     the stream read front to back with children_check and children_entry, as
 *                                 regk_read_children reads it: "0 <consumed> <skipped> <children> <err of every
 *                                 directory>", or "<code> <position> <directory>"
 * Results on stdout, whitespace separated.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../registrar_b200/csrc/regk_children.cuh"

using namespace regk;

int main()
{
    static char line[1 << 22];
    uint8_t *s = nullptr;
    uint64_t len = 0, d = 0;
    int32_t xb = 0;
    while (fgets(line, sizeof line, stdin)) {
        if (line[0] == 'S') {
            char *hex = strtok(line + 2, " \n");
            xb = (int32_t)strtol(strtok(nullptr, " \n"), nullptr, 10);
            d = strtoull(strtok(nullptr, " \n"), nullptr, 10);
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
                ChildHead h;
                printf("%u ", children_head(s + pos, len - pos, xb, d, &h));
            }
            printf("\n");
        } else if (line[0] == 'R') {
            uint64_t pos = strtoull(line + 2, nullptr, 10), k = 0, skipped = 0, children = 0;
            std::vector<int32_t> err;
            uint32_t code = CH_OK;
            uint64_t at = 0;
            while (k < d) {
                ChildHead h;
                code = children_check(s + pos, len - pos, xb, d, k, &h);
                at = pos;
                if (code != CH_OK)
                    break;
                const uint64_t end = pos + 4u + (uint32_t)h.len;
                if (h.kind == RK_REPLY) {
                    if (h.err == 0) {
                        uint64_t p = pos + 24;
                        for (int32_t i = 0; i < h.count && code == CH_OK; i++) {
                            uint32_t L;
                            code = children_entry(s + p, end - p, &L);
                            at = p;
                            p += 4u + L;
                            children++;
                        }
                        if (code == CH_OK && p != end) {
                            code = CH_ENT_END;
                            at = p;
                        }
                        if (code != CH_OK)
                            break;
                    }
                    err.push_back(h.err);
                    k++;
                } else {
                    skipped++;
                }
                pos = end;
            }
            if (code != CH_OK) {
                printf("%u %llu %llu\n", code, (unsigned long long)at, (unsigned long long)k);
            } else {
                printf("0 %llu %llu %llu", (unsigned long long)pos, (unsigned long long)skipped, (unsigned long long)children);
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
