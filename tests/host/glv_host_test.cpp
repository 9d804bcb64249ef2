// Host-side run of glv_decompose (csrc/glv.cuh, compiled with g++) over scalars written by tests/test_host_glv.py.
// In:  u64 n, then n x 8 u32 limbs of a canonical scalar k < r.
// Out: n x { 4 u32 |k1|, 4 u32 |k2|, u32 neg1, u32 neg2 }; the Python side checks k1 + lambda k2 = k (mod r) and the bounds.
#include <cstdio>
#include <cstdint>
#include <vector>
#include "../../distributed_groth16_b200/csrc/glv.cuh"

using namespace b200zk;

int main(int argc, char** argv) {
    if (argc < 3) { printf("usage: glv_host_test in.bin out.bin\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    if (!f) return 2;
    uint64_t n = 0;
    if (fread(&n, 8, 1, f) != 1) return 2;
    std::vector<uint32_t> in(n * 8), out(n * 10);
    if (fread(in.data(), 4, n * 8, f) != n * 8) return 2;
    fclose(f);
    for (uint64_t i = 0; i < n; ++i) {
        GlvSplit s = glv_decompose(&in[i * 8]);
        uint32_t* o = &out[i * 10];
        for (int j = 0; j < 4; ++j) { o[j] = s.k1[j]; o[4 + j] = s.k2[j]; }
        o[8] = s.neg1 ? 1u : 0u;
        o[9] = s.neg2 ? 1u : 0u;
    }
    FILE* g = fopen(argv[2], "wb");
    if (!g || fwrite(out.data(), 4, n * 10, g) != n * 10) return 2;
    fclose(g);
    printf("ALL OK %llu\n", (unsigned long long)n);
    return 0;
}
