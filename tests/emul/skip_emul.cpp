/*
 * skip_emul.cpp — TEST INFRASTRUCTURE: the skip-mode fence pass (regk_fence_kernel, regk_skip.cuh) on the CPU.
 * fence_record() of registrar_b200/csrc/regk_core.cuh is host+device code; compiled here with g++ it is compared
 * with the oracle's restatement of the fence by tests/test_skip_fence.py.  Not part of the product library.
 */
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/regk.h"
#include "../../registrar_b200/csrc/regk_core.cuh"

using namespace regk;

extern "C" {

/* The skip-mode fence pass (regk_fence_kernel) on the CPU: fence_record() per record, with the batch's flags, over
   word-padded copies of the byte arrays read through GuardedWords as the kernel does.  bits[n] out; returns the OR. */
uint32_t emul_fence(const regk_batch *b, uint32_t ntypes, uint8_t *bits)
{
    const bool alias = b->flags & REGK_NODE_ALIAS, do_path = !(b->flags & REGK_NO_PATH), do_json = !(b->flags & REGK_NO_JSON);
    const uint64_t n = b->n;
    auto words = [](const uint8_t *p, uint64_t len) {
        std::vector<uint32_t> w(len / 4 + 2, 0xA5A5A5A5u);
        if (len)
            memcpy(w.data(), p, len);
        return w;
    };
    const uint64_t host_len = alias ? 0 : (b->host_off ? b->host_off[n] : n * b->host_stride);
    const std::vector<uint32_t> dw = words(b->domain_bytes, n ? b->domain_off[n] : 0), hw = words(b->host_bytes, host_len),
                                aw = words(b->addr_bytes, n ? b->addr_off[n] : 0);
    uint32_t bad_all = 0;
    for (uint64_t r = 0; r < n; r++) {
        const uint32_t d0 = b->domain_off[r], L = b->domain_off[r + 1] - d0;
        const uint32_t h0 = alias ? 0 : (b->host_off ? b->host_off[r] : (uint32_t)(r * b->host_stride));
        const uint32_t H = alias ? 0 : (b->host_off ? b->host_off[r + 1] - b->host_off[r] : b->host_stride);
        const uint32_t a0 = b->addr_off[r], al = b->addr_off[r + 1] - a0;
        bits[r] = (uint8_t)fence_record(GuardedWords{dw.data()}, d0, L, GuardedWords{hw.data()}, h0, H, GuardedWords{aw.data()},
            a0, al, b->type_id[r], ntypes, alias, do_path, do_json);
        bad_all |= bits[r];
    }
    return bad_all;
}


}  /* extern "C" */
