/*
 * reconcile_emul.cpp — TEST INFRASTRUCTURE: the clamped string helpers of regk_core.cuh (word_clamped,
 * string_word_clamped, string_hash32_clamped, string_equal2), which regk_reconcile.cuh uses on a caller's snapshot
 * streams, on the CPU.  Built as a standalone program with -fsanitize=address,undefined by tests/test_reconcile.py:
 * every buffer is allocated with exactly its length, so a read past its end stops the program.  Not part of the
 * product library.
 *
 * stdin, one command per line (bytes in hex, "-" for none):
 *   A <hex>          buffer A: exactly these bytes          B <hex>   the same for buffer B
 *   W <o> <k>        string_word_clamped(A, o, k, |A|)      H <o> <n> string_hash32_clamped(A, o, n, |A|)
 *   E <a> <b> <n>    string_equal2(A, a, |A|, B, b, |B|, n)
 * One decimal result per W / H / E line on stdout.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "../../registrar_b200/csrc/regk_core.cuh"

using namespace regk;

static uint8_t *load(const char *hex, uint64_t *len)
{
    const size_t h = strcmp(hex, "-") ? strlen(hex) : 0;
    *len = h / 2;
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
    uint8_t *A = nullptr, *B = nullptr;
    uint64_t la = 0, lb = 0;
    while (fgets(line, sizeof line, stdin)) {
        char cmd = line[0];
        if (cmd == 'A' || cmd == 'B') {
            char *hex = line + 2;
            hex[strcspn(hex, "\r\n")] = 0;
            uint8_t *&buf = cmd == 'A' ? A : B;
            free(buf);
            buf = load(hex, cmd == 'A' ? &la : &lb);
        } else if (cmd == 'W') {
            unsigned long long o, k;
            sscanf(line + 2, "%llu %llu", &o, &k);
            printf("%u\n", string_word_clamped(reinterpret_cast<const uint32_t *>(A), o, (uint32_t)k, la));
        } else if (cmd == 'H') {
            unsigned long long o, n;
            sscanf(line + 2, "%llu %llu", &o, &n);
            printf("%u\n", string_hash32_clamped(reinterpret_cast<const uint32_t *>(A), o, (uint32_t)n, la));
        } else if (cmd == 'E') {
            unsigned long long a, b, n;
            sscanf(line + 2, "%llu %llu %llu", &a, &b, &n);
            printf("%d\n", string_equal2(reinterpret_cast<const uint32_t *>(A), a, la, reinterpret_cast<const uint32_t *>(B), b,
                                         lb, (uint32_t)n) ? 1 : 0);
        }
    }
    free(A);
    free(B);
    return 0;
}
