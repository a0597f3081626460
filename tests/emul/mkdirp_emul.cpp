/*
 * mkdirp_emul.cpp — TEST INFRASTRUCTURE: the per-directory helpers of regk_mkdirp.cuh on the CPU.
 * mkdir_components() and mkdir_extend() of registrar_b200/csrc/regk_core.cuh are host+device code; compiled here with
 * g++ they are compared with the restatement in tests/mkdirp_util.py by tests/test_mkdirp_set.py.  Not part of the
 * product library.
 */
#include <cstdint>
#include <cstring>

#include "../../registrar_b200/csrc/regk_core.cuh"

using namespace regk;

extern "C" {

/* Packed directories d_k = bytes[off[k], off[k+1]): comps[k] = mkdir_components(d_k) (MKDIR_INVALID as 0xFFFFFFFF);
   for the valid ones, the prefix ends the kernels' depth loop visits, written from ends[ends_off[k]] on, and the
   slot hash of each (hashes[]).  Returns the number of ends written. */
uint64_t emul_mkdirp(const uint8_t *bytes, const uint64_t *off, uint64_t n, uint32_t *comps, uint32_t *ends, uint32_t *hashes)
{
    uint64_t w = 0;
    for (uint64_t k = 0; k < n; k++) {
        const uint8_t *p = bytes + off[k];
        const uint32_t L = (uint32_t)(off[k + 1] - off[k]);
        const uint32_t c = mkdir_components(p, L);
        comps[k] = c;
        if (c == MKDIR_INVALID || c == 0)
            continue;
        uint32_t pos = 0, h = MKDIR_HASH_SEED;
        do {
            pos = mkdir_extend(p, pos, L, &h);
            ends[w] = pos;
            hashes[w] = mkdir_slot_hash(h, pos);
            w++;
        } while (pos < L);
    }
    return w;
}

}  /* extern "C" */
