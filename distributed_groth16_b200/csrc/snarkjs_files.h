// snarkjs_files.h -- the host side of snarkjs's binary files and JSON output, for the native prover (zkey.cu,
// b200zk_zkey_*): the section table of a .zkey / .wtns, the Groth16 zkey header and the wtns header with the checks
// formats.read_zkey / read_wtns make (same message text), and the proof.json / public.json writer of
// formats.write_proof_json / write_public_json (JSON.stringify(obj, null, 1): one-space indent, no trailing newline).
// Plain C++17 without CUDA, so that tests/host/snarkjs_files_host_test.cpp builds it with g++; the record predicate is also
// compiled for the device.
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>

#ifdef __CUDACC__
#define SJF_HD __host__ __device__ __forceinline__
#else
#define SJF_HD inline
#endif

namespace b200zk {
namespace sjf {

// little-endian u64 limbs of the BN254 base field q and scalar field r
static const uint64_t FQ_LE[4] = {0x3c208c16d87cfd47ull, 0x97816a916871ca8dull, 0xb85045b68181585dull, 0x30644e72e131a029ull};
static const uint64_t FR_LE[4] = {0x43e1f593f0000001ull, 0x2833e84879b97091ull, 0xb85045b68181585dull, 0x30644e72e131a029ull};

inline uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }

inline bool eq_le(const uint8_t* p, const uint64_t want[4]) {
    for (int i = 0; i < 4; ++i) if (rd64(p + 8 * i) != want[i]) return false;
    return true;
}

// 32 little-endian bytes < r
inline bool below_r(const uint8_t* p) {
    for (int i = 3; i >= 0; --i) {
        const uint64_t v = rd64(p + 8 * i);
        if (v != FR_LE[i]) return v < FR_LE[i];
    }
    return false;
}

// A coefficient record (matrix m, constraint c, signal s) the QAP can index: A or B, a variable of the key, a row of the domain.
SJF_HD bool coef_record_ok(uint32_t m, uint32_t c, uint32_t s, uint32_t n_vars, uint32_t domain_size) {
    return m <= 1 && s < n_vars && c < domain_size;
}

// Python's repr() of a bytes object (the "bad magic" message quotes it as formats._sections does)
inline std::string py_bytes_repr(const uint8_t* p, size_t n) {
    bool sq = false, dq = false;
    for (size_t i = 0; i < n; ++i) { sq |= p[i] == '\''; dq |= p[i] == '"'; }
    const char quote = sq && !dq ? '"' : '\'';
    std::string s = "b";
    s += quote;
    for (size_t i = 0; i < n; ++i) {
        const uint8_t c = p[i];
        char b[8];
        if (c == (uint8_t)quote || c == '\\') { s += '\\'; s += (char)c; }
        else if (c == '\t') s += "\\t";
        else if (c == '\n') s += "\\n";
        else if (c == '\r') s += "\\r";
        else if (c < 0x20 || c >= 0x7f) { snprintf(b, sizeof(b), "\\x%02x", c); s += b; }
        else s += (char)c;
    }
    s += quote;
    return s;
}

// ---- section table ------------------------------------------------------------------------------------------------------
// magic (4) | version u32 | n_sections u32 | n_sections x (id u32, length u64, payload).  Only the first section of an id is
// kept, as formats._sections uses it.  Every section must lie inside the buffer.
struct Sections {
    static const uint32_t MAX_ID = 16;
    uint64_t off[MAX_ID] = {}, len[MAX_ID] = {};
    bool has[MAX_ID] = {};
};

inline bool parse_sections(const uint8_t* buf, size_t n, const char magic[4], const char* kind, Sections* out, std::string* err) {
    if (n < 4 || memcmp(buf, magic, 4) != 0) {
        *err = "bad magic " + py_bytes_repr(buf, n < 4 ? n : 4) + " (expected " + py_bytes_repr((const uint8_t*)magic, 4) + ")";
        return false;
    }
    char b[192];
    if (n < 12) {
        snprintf(b, sizeof(b), "%s file of %zu bytes ends inside its header", kind, n);
        *err = b;
        return false;
    }
    const uint32_t nsec = rd32(buf + 8);
    uint64_t off = 12;
    for (uint32_t k = 0; k < nsec; ++k) {
        if (n - off < 12) {
            snprintf(b, sizeof(b), "%s section table runs past the end of the file (section %u of %u at byte %llu of %zu)", kind, k,
                     nsec, (unsigned long long)off, n);
            *err = b;
            return false;
        }
        const uint32_t sid = rd32(buf + off);
        const uint64_t ln = rd64(buf + off + 4);
        off += 12;
        if (ln > n - off) {
            snprintf(b, sizeof(b), "%s section %u runs past the end of the file (%llu + %llu > %zu bytes)", kind, sid,
                     (unsigned long long)off, (unsigned long long)ln, n);
            *err = b;
            return false;
        }
        if (sid < Sections::MAX_ID && !out->has[sid]) {
            out->has[sid] = true;
            out->off[sid] = off;
            out->len[sid] = ln;
        }
        off += ln;
    }
    return true;
}

// ---- Groth16 zkey ---------------------------------------------------------------------------------------------------------
struct Zkey {
    uint32_t n_vars = 0, n_public = 0, domain_size = 0, n_coef = 0;
    uint64_t hdr_points = 0;            // alpha_1 beta_1 beta_2 gamma_2 delta_1 delta_2 (64 64 128 128 64 128 bytes)
    uint64_t coef = 0;                  // the n_coef 44-byte records of section 4
    uint64_t ic = 0, a = 0, b1 = 0, b2 = 0, l = 0, h = 0;    // sections 3, 5, 6, 7, 8, 9
};

inline bool parse_zkey(const uint8_t* buf, size_t n, Zkey* z, std::string* err) {
    Sections s;
    if (!parse_sections(buf, n, "zkey", "zkey", &s, err)) return false;
    char b[192];
    for (uint32_t sid = 2; sid <= 9; ++sid)
        if (!s.has[sid]) { snprintf(b, sizeof(b), "zkey section %u missing", sid); *err = b; return false; }
    if (!s.has[1]) { *err = "zkey section 1 missing"; return false; }
    if (s.len[1] < 4) { *err = "zkey section 1 too short"; return false; }
    const uint32_t protocol = rd32(buf + s.off[1]);
    if (protocol != 1) {
        snprintf(b, sizeof(b), "zkey protocol %u is not Groth16 (1): PLONK (2) and FFLONK (10) keys are not supported", protocol);
        *err = b;
        return false;
    }
    // section 2: n8q q n8r r n_vars n_public domain_size, then the six vk points
    const uint8_t* h = buf + s.off[2];
    const uint64_t l2 = s.len[2];
    if (l2 < 4 || rd32(h) != 32 || l2 < 40 || !eq_le(h + 4, FQ_LE) || l2 < 44 || rd32(h + 36) != 32 || l2 < 72 || !eq_le(h + 40, FR_LE)) {
        *err = "zkey is not over BN254";
        return false;
    }
    if (l2 < 84 + 576) { *err = "zkey section 2 too short"; return false; }
    z->n_vars = rd32(h + 72);
    z->n_public = rd32(h + 76);
    z->domain_size = rd32(h + 80);
    z->hdr_points = s.off[2] + 84;
    if (z->n_vars == 0 || (uint64_t)z->n_public + 1 > z->n_vars) {
        snprintf(b, sizeof(b), "zkey header: n_public + 1 = %llu variables are public but n_vars = %u",
                 (unsigned long long)z->n_public + 1, z->n_vars);
        *err = b;
        return false;
    }
    if (z->domain_size == 0 || (z->domain_size & (z->domain_size - 1))) {
        snprintf(b, sizeof(b), "zkey header: domain size %u is not a power of two", z->domain_size);
        *err = b;
        return false;
    }
    if (s.len[4] < 4) { *err = "zkey section 4 too short"; return false; }
    z->n_coef = rd32(buf + s.off[4]);
    if (s.len[4] < 4 + (uint64_t)z->n_coef * 44) {
        snprintf(b, sizeof(b), "zkey coefficient section too short for %u records", z->n_coef);
        *err = b;
        return false;
    }
    z->coef = s.off[4] + 4;
    const uint64_t nv = z->n_vars, np1 = (uint64_t)z->n_public + 1;
    const struct { uint32_t sid; uint64_t bytes; uint64_t* dst; } need[6] = {
        {3, np1 * 64, &z->ic}, {5, nv * 64, &z->a}, {6, nv * 64, &z->b1}, {7, nv * 128, &z->b2}, {8, (nv - np1) * 64, &z->l},
        {9, (uint64_t)z->domain_size * 64, &z->h}};
    for (const auto& q : need) {
        if (s.len[q.sid] < q.bytes) { snprintf(b, sizeof(b), "zkey section %u too short", q.sid); *err = b; return false; }
        *q.dst = s.off[q.sid];
    }
    return true;
}

// ---- wtns ---------------------------------------------------------------------------------------------------------------
struct Wtns {
    uint32_t n = 0;
    uint64_t data = 0;                  // n x 32 bytes, canonical little-endian
};

inline bool parse_wtns(const uint8_t* buf, size_t len, Wtns* w, std::string* err) {
    Sections s;
    if (!parse_sections(buf, len, "wtns", "wtns", &s, err)) return false;
    if (!s.has[1]) { *err = "wtns section 1 missing"; return false; }
    const uint8_t* h = buf + s.off[1];
    const uint64_t l1 = s.len[1];
    if (l1 < 4 || rd32(h) != 32 || l1 < 36 || !eq_le(h + 4, FR_LE)) { *err = "wtns is not over BN254 Fr"; return false; }
    if (l1 < 40) { *err = "wtns section 1 too short"; return false; }
    w->n = rd32(h + 36);
    if (!s.has[2]) { *err = "wtns section 2 missing"; return false; }
    if (s.len[2] < (uint64_t)w->n * 32) { *err = "wtns data section too short"; return false; }
    w->data = s.off[2];
    return true;
}

// ---- decimals and JSON ----------------------------------------------------------------------------------------------------
// a 256-bit integer (4 little-endian u64 limbs) in decimal
inline std::string dec(const uint64_t le[4]) {
    uint64_t x[4] = {le[0], le[1], le[2], le[3]};
    const uint64_t BASE = 10000000000000000000ull;       // 10^19
    uint64_t parts[5];                                   // 2^256 < 10^(5 * 19)
    int np = 0;
    while (x[0] | x[1] | x[2] | x[3]) {
        unsigned __int128 rem = 0;
        for (int i = 3; i >= 0; --i) {
            const unsigned __int128 cur = (rem << 64) | x[i];
            x[i] = (uint64_t)(cur / BASE);
            rem = cur % BASE;
        }
        parts[np++] = (uint64_t)rem;
    }
    if (np == 0) return "0";
    char b[96];
    int o = snprintf(b, sizeof(b), "%llu", (unsigned long long)parts[np - 1]);
    for (int i = np - 2; i >= 0; --i) o += snprintf(b + o, sizeof(b) - o, "%019llu", (unsigned long long)parts[i]);
    return std::string(b, o);
}

inline std::string dec_le(const uint8_t* p) {
    uint64_t v[4];
    for (int i = 0; i < 4; ++i) v[i] = rd64(p + 8 * i);
    return dec(v);
}

inline std::string dec_be(const uint8_t* p) {
    uint64_t v[4] = {0, 0, 0, 0};
    for (int i = 0; i < 32; ++i) v[(31 - i) / 8] |= (uint64_t)p[i] << (8 * ((31 - i) % 8));
    return dec(v);
}

// ffjavascript's uncompressed encodings (b200zk_points_encode_dev fmt 0): G1 x || y, G2 x.c1 x.c0 y.c1 y.c0, big-endian;
// infinity has 0x40 in byte 0
inline std::string g1_json(const uint8_t* e, const char* ind) {
    const std::string i1 = std::string(ind) + " ";
    if (e[0] & 0x40) return "[\n" + i1 + "\"0\",\n" + i1 + "\"1\",\n" + i1 + "\"0\"\n" + ind + "]";
    return "[\n" + i1 + "\"" + dec_be(e) + "\",\n" + i1 + "\"" + dec_be(e + 32) + "\",\n" + i1 + "\"1\"\n" + ind + "]";
}

inline std::string g2_json(const uint8_t* e, const char* ind) {
    const std::string i1 = std::string(ind) + " ", i2 = i1 + " ";
    auto pair = [&](const std::string& c0, const std::string& c1) {
        return "[\n" + i2 + "\"" + c0 + "\",\n" + i2 + "\"" + c1 + "\"\n" + i1 + "]";
    };
    if (e[0] & 0x40) return "[\n" + i1 + pair("0", "0") + ",\n" + i1 + pair("1", "0") + ",\n" + i1 + pair("0", "0") + "\n" + ind + "]";
    return "[\n" + i1 + pair(dec_be(e + 32), dec_be(e)) + ",\n" + i1 + pair(dec_be(e + 96), dec_be(e + 64)) + ",\n" + i1 +
           pair("1", "0") + "\n" + ind + "]";
}

// snarkjs's proof.json from the encodings of A (64 bytes), B (128) and C (64)
inline std::string proof_json(const uint8_t* a, const uint8_t* b, const uint8_t* c) {
    return "{\n \"pi_a\": " + g1_json(a, " ") + ",\n \"pi_b\": " + g2_json(b, " ") + ",\n \"pi_c\": " + g1_json(c, " ") +
           ",\n \"protocol\": \"groth16\",\n \"curve\": \"bn128\"\n}";
}

// snarkjs's public.json from n canonical little-endian 32-byte values
inline std::string public_json(const uint8_t* le, size_t n) {
    if (n == 0) return "[]";
    std::string s = "[";
    for (size_t i = 0; i < n; ++i) s += (i ? ",\n \"" : "\n \"") + dec_le(le + 32 * i) + "\"";
    return s + "\n]";
}

}  // namespace sjf
}  // namespace b200zk
