/*
 * results_emul.cpp — TEST INFRASTRUCTURE: the per-frame and per-entry helpers of regk_results.cuh (results_head,
 * results_check, results_entry) on the CPU.  Built as a standalone program with -fsanitize=address,undefined by
 * tests/test_results_cpu.py: the stream and the framed paths are allocated with exactly their lengths, so a read past
 * their end stops the program.  Not part of the product library.
 *
 * stdin, one command per line:
 *   S <hex or ->                                        the stream
 *   F <xid_base> <op> <group> <multi> <tol> <n> <path hex>:<data length> ...   the framing (group >= 1)
 *   P                                                   results_head at every position: one code per position
 *   R <start>                                           the stream read front to back with results_check and, for
 *                                                       every reply, results_entry of its entries in order, as
 *                                                       regk_read_results reads it: "0 <consumed> <skipped> <frame
 *                                                       errs...> | <err cls version of every entry...>", or "<code>
 *                                                       <position> <frame>"
 * Results on stdout, whitespace separated.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../registrar_b200/csrc/regk_results.cuh"

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
    uint8_t *s = nullptr, *paths = nullptr;
    uint64_t len = 0;
    std::vector<unsigned long long> poff, doff;
    ResFraming f{};
    int32_t tol = 0;
    while (fgets(line, sizeof line, stdin)) {
        if (line[0] == 'S') {
            free(s);
            s = unhex(strtok(line + 2, " \n"), &len);
        } else if (line[0] == 'F') {
            f = ResFraming{};
            f.xid_base = (int32_t)strtol(strtok(line + 2, " \n"), nullptr, 10);
            f.op = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            f.group = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            f.multi = (uint32_t)strtoul(strtok(nullptr, " \n"), nullptr, 10);
            tol = (int32_t)strtol(strtok(nullptr, " \n"), nullptr, 10);
            f.entries = strtoull(strtok(nullptr, " \n"), nullptr, 10);
            f.frames = (f.entries + f.group - 1) / f.group;
            std::vector<uint8_t> all;
            poff.assign(1, 0);
            doff.assign(1, 0);
            for (uint64_t e = 0; e < f.entries; e++) {
                char *tok = strtok(nullptr, " \n");
                char *colon = strchr(tok, ':');
                *colon = 0;
                uint64_t pl;
                uint8_t *p = unhex(tok, &pl);
                all.insert(all.end(), p, p + pl);
                free(p);
                poff.push_back(all.size());
                doff.push_back(doff.back() + strtoull(colon + 1, nullptr, 10));
            }
            free(paths);
            paths = (uint8_t *)malloc(all.size() ? all.size() : 1);
            if (!all.empty())
                memcpy(paths, all.data(), all.size());
            f.path_bytes = paths;
            f.path_off = poff.data();
            f.data_off = doff.data();
        } else if (line[0] == 'P') {
            for (uint64_t pos = 0; pos < len; pos++) {
                ResHead h;
                printf("%u ", results_head(s + pos, len - pos, f, &h));
            }
            printf("\n");
        } else if (line[0] == 'R') {
            uint64_t pos = strtoull(line + 2, nullptr, 10), k = 0, skipped = 0;
            std::vector<int32_t> ferr;
            std::vector<ResEntry> ents;
            uint32_t code = RS_OK;
            uint64_t at = 0;
            while (k < f.frames) {
                ResHead h;
                code = results_check(s + pos, len - pos, f, k, &h);
                at = pos;
                if (code != RS_OK)
                    break;
                if (h.kind == RK_REPLY) {
                    const uint64_t a = k * f.group, b = a + f.group < f.entries ? a + f.group : f.entries;
                    for (uint64_t e = a; e < b && code == RS_OK; e++) {
                        ResEntry r;
                        code = results_entry(s, pos, f, k, e, tol, &r);
                        at = r.at;
                        ents.push_back(r);
                    }
                    if (code != RS_OK)
                        break;
                    ferr.push_back(h.err);
                    k++;
                } else {
                    skipped++;
                }
                pos += 4u + (uint32_t)h.len;
            }
            if (code != RS_OK) {
                printf("%u %llu %llu\n", code, (unsigned long long)at, (unsigned long long)k);
            } else {
                printf("0 %llu %llu", (unsigned long long)pos, (unsigned long long)skipped);
                for (int32_t e : ferr)
                    printf(" %d", e);
                printf(" |");
                for (const ResEntry &r : ents)
                    printf(" %d %u %d", r.err, (unsigned)r.cls, r.version);
                printf("\n");
            }
        }
        fflush(stdout);
    }
    free(s);
    free(paths);
    return 0;
}
