/*
 * regk_types.hpp — host-side construction of the per-type JSON fragment table
 * consumed by regk_json_kernel (and by the CPU logic tests).
 *
 * For every record type T (registration.type, lib/register.js:142) two byte
 * strings are precomputed, JSON-escaped once (ECMA-262 QuoteJSONString):
 *     f1 = {"type":"T","address":"          f2 = ,"T":{"address":"
 * Blob layout: TypeFrag[ntypes] (padded to 16 bytes) followed by the fragments.  Every
 * fragment is stored four times, pre-shifted by 0..3 zero bytes and zero padded to
 * frag_stride_words(len) words, so the kernel can append it at any byte phase of the
 * output with plain word copies; total size padded to 16 bytes.
 */
#ifndef REGK_TYPES_HPP
#define REGK_TYPES_HPP

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "regk_core.cuh"

namespace regk {

/* ECMA-262 QuoteJSONString without the surrounding quotes. */
inline std::string json_escape(const std::string &s)
{
    static const char hex[] = "0123456789abcdef";
    std::string o;
    for (unsigned char c : s) {
        switch (c) {
        case '"': o += "\\\""; break;
        case '\\': o += "\\\\"; break;
        case '\b': o += "\\b"; break;
        case '\f': o += "\\f"; break;
        case '\n': o += "\\n"; break;
        case '\r': o += "\\r"; break;
        case '\t': o += "\\t"; break;
        default:
            if (c < 0x20) {
                o += "\\u00";
                o += hex[c >> 4];
                o += hex[c & 15];
            } else {
                o += (char)c;
            }
        }
    }
    return o;
}

/* V8 enumerates "array index" keys (canonical decimal strings < 2^32 - 1) before string keys. */
inline bool is_array_index(const std::string &s)
{
    if (s.empty() || s.size() > 10)
        return false;
    if (s.size() > 1 && s[0] == '0')
        return false;
    unsigned long long v = 0;
    for (char c : s) {
        if (c < '0' || c > '9')
            return false;
        v = v * 10 + (unsigned)(c - '0');
    }
    return v < 4294967295ull;
}

/* Well-formed UTF-8 (Unicode table 3-7): no overlong form, no encoded surrogate D800-DFFF, nothing above
   U+10FFFF, no truncated sequence and no stray continuation byte.  Only such bytes are the UTF-8 form of a JS
   string, so only they can be a type the reference writes; the composers copy bytes >= 0x80 unchanged. */
inline bool utf8_well_formed(const std::string &s)
{
    const size_t n = s.size();
    size_t i = 0;
    while (i < n) {
        const unsigned c = (unsigned char)s[i];
        if (c < 0x80) {
            i++;
            continue;
        }
        size_t len;
        unsigned lo = 0x80, hi = 0xBF;                      /* range of the second byte */
        if (c >= 0xC2 && c <= 0xDF) {
            len = 2;
        } else if (c >= 0xE0 && c <= 0xEF) {
            len = 3;
            lo = c == 0xE0 ? 0xA0 : 0x80;                   /* E0 80..9F: overlong */
            hi = c == 0xED ? 0x9F : 0xBF;                   /* ED A0..BF: surrogates */
        } else if (c >= 0xF0 && c <= 0xF4) {
            len = 4;
            lo = c == 0xF0 ? 0x90 : 0x80;                   /* F0 80..8F: overlong */
            hi = c == 0xF4 ? 0x8F : 0xBF;                   /* F4 90..BF: above U+10FFFF */
        } else {
            return false;                                   /* continuation byte, C0 / C1, F5..FF */
        }
        if (n - i < len)
            return false;
        const unsigned c1 = (unsigned char)s[i + 1];
        if (c1 < lo || c1 > hi)
            return false;
        for (size_t k = 2; k < len; k++)
            if (((unsigned char)s[i + k] & 0xC0) != 0x80)
                return false;
        i += len;
    }
    return true;
}

constexpr size_t TYPE_BLOB_MAX = 16384;

/* Returns 0 on success, 1 = out-of-domain type name, 2 = table too large; *err gets the reason. */
inline int build_type_blob(const std::vector<std::string> &types, std::vector<uint8_t> *blob, uint32_t *max_escaped,
    std::string *err)
{
    const size_t ntypes = types.size();
    std::vector<TypeFrag> frags(ntypes);
    std::vector<uint8_t> bytes;
    const size_t table = (sizeof(TypeFrag) * std::max<size_t>(ntypes, 1) + 15) & ~(size_t)15;
    uint32_t maxq = 0;
    for (size_t i = 0; i < ntypes; i++) {
        const std::string &t = types[i];
        /* lib/register.js:152 `_obj[type] = {...}`: these names would overwrite a fixed key in place, and
           array-index names are enumerated first by V8 — both change the byte layout.  "__proto__" assigns the
           object's prototype instead of creating an own property, so JSON.stringify drops the nested object. */
        if (t == "type" || t == "address" || t == "ttl" || t == "__proto__" || is_array_index(t)) {
            *err = "type '" + t + "' collides with a fixed key, is an array index or is __proto__";
            return 1;
        }
        if (!utf8_well_formed(t)) {
            *err = "type " + std::to_string(i) + " is not well-formed UTF-8";
            return 1;
        }
        const std::string q = json_escape(t);
        maxq = std::max<uint32_t>(maxq, (uint32_t)q.size());
        const std::string f1 = "{\"type\":\"" + q + "\",\"address\":\"";
        const std::string f2 = ",\"" + q + "\":{\"address\":\"";
        auto add = [&](const std::string &f, uint16_t &off, uint16_t &len) {
            while (bytes.size() % 4)
                bytes.push_back(0);
            off = (uint16_t)(table + bytes.size());
            len = (uint16_t)f.size();
            const size_t stride = frag_stride_words((uint32_t)f.size()) * 4;
            for (size_t shift = 0; shift < 4; shift++) {
                const size_t start = bytes.size();
                bytes.insert(bytes.end(), shift, 0);
                bytes.insert(bytes.end(), f.begin(), f.end());
                bytes.resize(start + stride, 0);
            }
        };
        if (table + bytes.size() + 4 * (f1.size() + f2.size() + 16) > TYPE_BLOB_MAX) {
            *err = "fragment table exceeds the shared-memory budget of 16384 bytes";
            return 2;
        }
        add(f1, frags[i].f1_off, frags[i].f1_len);
        add(f2, frags[i].f2_off, frags[i].f2_len);
    }
    blob->assign((table + bytes.size() + 4 + 15) & ~(size_t)15, 0);
    if (ntypes)
        memcpy(blob->data(), frags.data(), sizeof(TypeFrag) * ntypes);
    if (!bytes.empty())
        memcpy(blob->data() + table, bytes.data(), bytes.size());
    *max_escaped = maxq;
    return 0;
}

}  // namespace regk
#endif
