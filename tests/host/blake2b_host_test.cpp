// csrc/blake2b.cuh on the host: the RFC 7693 Appendix A vector, digests that do not depend on how the input is split,
// the lazy buffer rule as it shows in the exported state, and export / import round trips.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../distributed_groth16_b200/csrc/blake2b.cuh"

using namespace b200zk;

static int fails = 0;
#define CHECK(c, ...)                        \
    do {                                     \
        if (!(c)) {                          \
            printf("FAIL: " __VA_ARGS__);    \
            printf("\n");                    \
            ++fails;                         \
        }                                    \
    } while (0)

static void digest(const std::vector<uint8_t>& in, const std::vector<size_t>& cuts, uint8_t out[64]) {
    blake2b_ctx c;
    blake2b_init(&c, 64);
    size_t lo = 0;
    for (size_t hi : cuts) {
        blake2b_update(&c, in.data() + lo, hi - lo);
        lo = hi;
    }
    blake2b_update(&c, in.data() + lo, in.size() - lo);
    blake2b_final(&c, out);
}

static uint64_t rd64(const uint8_t* p) {
    uint64_t v = 0;
    for (int k = 7; k >= 0; --k) v = (v << 8) | p[k];
    return v;
}
static uint32_t rd32(const uint8_t* p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }

int main() {
    // RFC 7693 Appendix A: BLAKE2b-512("abc")
    static const uint8_t abc[64] = {
        0xBA, 0x80, 0xA5, 0x3F, 0x98, 0x1C, 0x4D, 0x0D, 0x6A, 0x27, 0x97, 0xB6, 0x9F, 0x12, 0xF6, 0xE9,
        0x4C, 0x21, 0x2F, 0x14, 0x68, 0x5A, 0xC4, 0xB7, 0x4B, 0x12, 0xBB, 0x6F, 0xDB, 0xFF, 0xA2, 0xD1,
        0x7D, 0x87, 0xC5, 0x39, 0x2A, 0xAB, 0x79, 0x2D, 0xC2, 0x52, 0xD5, 0xDE, 0x45, 0x33, 0xCC, 0x95,
        0x18, 0xD3, 0x8A, 0xA8, 0xDB, 0xF1, 0x92, 0x5A, 0xB9, 0x23, 0x86, 0xED, 0xD4, 0x00, 0x99, 0x23};
    uint8_t out[64], ref[64];
    digest(std::vector<uint8_t>{'a', 'b', 'c'}, {}, out);
    CHECK(memcmp(out, abc, 64) == 0, "RFC 7693 Appendix A vector");

    srand(7);
    for (size_t len : {0, 1, 127, 128, 129, 255, 256, 257, 1000, 4096, 65537}) {
        std::vector<uint8_t> in(len);
        for (auto& b : in) b = (uint8_t)rand();
        digest(in, {}, ref);
        for (int trial = 0; trial < 20; ++trial) {
            std::vector<size_t> cuts;
            size_t at = 0;
            while (len && at < len && cuts.size() < 40) {
                at += (size_t)rand() % (trial < 10 ? 8 : 300);
                if (at <= len) cuts.push_back(at);
            }
            digest(in, cuts, out);
            CHECK(memcmp(out, ref, 64) == 0, "digest of %zu bytes depends on the split (trial %d)", len, trial);
        }
        // export after every cut, import, continue: the same digest
        blake2b_ctx c;
        blake2b_init(&c, 64);
        size_t lo = 0;
        while (lo < len) {
            const size_t step = 1 + (size_t)rand() % 200;
            const size_t hi = lo + step < len ? lo + step : len;
            uint8_t st[BLAKE2B_STATE_BYTES];
            blake2b_export(&c, st);
            blake2b_ctx d;
            CHECK(blake2b_import(&d, st), "import of an exported state");
            blake2b_update(&d, in.data() + lo, hi - lo);
            c = d;
            lo = hi;
        }
        blake2b_final(&c, out);
        CHECK(memcmp(out, ref, 64) == 0, "export / import round trip over %zu bytes", len);
    }

    // the lazy rule: after exactly 128 k bytes the k-th block is still buffered, uncompressed and not counted
    for (size_t k = 1; k <= 4; ++k) {
        std::vector<uint8_t> in(128 * k, 0x5A);
        blake2b_ctx c;
        blake2b_init(&c, 64);
        blake2b_update(&c, in.data(), in.size());
        uint8_t st[BLAKE2B_STATE_BYTES];
        blake2b_export(&c, st);
        CHECK(rd32(st + 208) == 128, "c after %zu blocks = %u", k, rd32(st + 208));
        CHECK(rd64(st + 192) == 128 * (k - 1) && rd64(st + 200) == 0, "t after %zu blocks", k);
        CHECK(rd32(st + 212) == 64, "outlen in the state");
        CHECK(memcmp(st, in.data(), 128) == 0, "the last block stays in the buffer");
        if (k == 1) {
            blake2b_ctx fresh;
            blake2b_init(&fresh, 64);
            uint8_t st0[BLAKE2B_STATE_BYTES];
            blake2b_export(&fresh, st0);
            CHECK(memcmp(st0 + 128, st + 128, 64) == 0, "h unchanged after one full block");
        }
    }
    uint8_t bad[BLAKE2B_STATE_BYTES] = {0};
    blake2b_ctx d;
    CHECK(!blake2b_import(&d, bad), "a state with outlen 0 is refused");

    if (fails) {
        printf("%d failures\n", fails);
        return 1;
    }
    printf("ALL OK\n");
    return 0;
}
