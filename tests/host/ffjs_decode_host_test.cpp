// Host-side check of the ffjavascript decoder in csrc/codec.cuh (ffjs_get / ffjs_decode, g++, PTX carry primitives
// emulated) against vectors written by the Python oracle.
// File: u64 n, then n x { u32 g2, u32 compressed, u32 check_subgroup, u32 valid, 128 B encoding (zero-padded),
//                         16 u64 expected affine (Montgomery, zero-padded) }.
#include <cstdio>
#include <cstring>
#include <cstdint>
#include "../../distributed_groth16_b200/csrc/codec.cuh"

using namespace b200zk;

template <class F, bool C>
static int check_one(uint64_t i, const uint8_t* enc, bool sub, bool valid, const uint64_t* exp) {
    constexpr int LEN = (C ? 1 : 2) * (int)sizeof(F);
    affine_t<F> p;
    const bool ok = ffjs_decode<F, C>(enc, sub, &p);
    if (ok != valid) { printf("case %llu: validity %d, want %d\n", (unsigned long long)i, ok, valid); return 1; }
    if (!ok) {
        if (!p.is_inf()) { printf("case %llu: invalid slot not infinity\n", (unsigned long long)i); return 1; }
        return 0;
    }
    if (memcmp(&p, exp, sizeof(p))) { printf("case %llu: point mismatch\n", (unsigned long long)i); return 1; }
    uint8_t back[LEN];
    ffjs_encode<F, C>(p, back);
    if (memcmp(back, enc, LEN)) { printf("case %llu: re-encoding mismatch\n", (unsigned long long)i); return 1; }
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    uint64_t n = 0;
    if (fread(&n, 8, 1, f) != 1) return 2;
    int fails = 0;
    for (uint64_t i = 0; i < n; ++i) {
        uint32_t hdr[4];
        uint8_t enc[128];
        uint64_t exp[16];
        if (fread(hdr, 4, 4, f) != 4 || fread(enc, 1, 128, f) != 128 || fread(exp, 8, 16, f) != 16) return 2;
        const bool g2 = hdr[0] != 0, c = hdr[1] != 0, sub = hdr[2] != 0, valid = hdr[3] != 0;
        if (g2) fails += c ? check_one<Fq2, true>(i, enc, sub, valid, exp) : check_one<Fq2, false>(i, enc, sub, valid, exp);
        else fails += c ? check_one<Fq, true>(i, enc, sub, valid, exp) : check_one<Fq, false>(i, enc, sub, valid, exp);
    }
    fclose(f);
    printf(fails ? "FAILED %d of %llu\n" : "ALL OK %d of %llu\n", fails, (unsigned long long)n);
    return fails ? 1 : 0;
}
