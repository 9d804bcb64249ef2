// Host-side run of b200zk_test_arith's op bodies (csrc/selftest.cu's arith_apply<OP>, compiled with g++: PTX carry primitives
// emulated) over records written by tests/test_host_arith.py.
// In:  u64 block count, then per block u64 op, u64 n, u64 in_words, then n x in_words u64.
// Out: per block n x out_words u64 (the op's record size); the Python side compares them with the big-integer answers.
// Device-only ops (fr_root_of_unity, quad_ops) are refused.  Prints ALL OK on success.
// `arith_host_test --table` prints "op in out" for every op arith_words knows, device-only ones included.
#include <cstdio>
#include <cstdint>
#include <string>
#include <vector>
#include "../../distributed_groth16_b200/csrc/selftest.cu"

using namespace b200zk;

static bool run(int op, const uint64_t* in, uint64_t* out, size_t n, int in_w, int out_w) {
    switch (op) {
#define B2_ARITH_HOST_CASE(OP, IN, OUT) \
        case OP: for (size_t i = 0; i < n; ++i) arith_apply<OP>(in + i * in_w, out + i * out_w); return true;
        B2_ARITH_OPS(B2_ARITH_HOST_CASE)
#undef B2_ARITH_HOST_CASE
        default: return false;
    }
}

int main(int argc, char** argv) {
    if (argc == 2 && std::string(argv[1]) == "--table") {
        for (int op = 0; op < 256; ++op) {
            int in_w, out_w;
            arith_words(op, &in_w, &out_w);
            if (in_w) printf("%d %d %d\n", op, in_w, out_w);
        }
        return 0;
    }
    if (argc < 3) { printf("usage: arith_host_test in.bin out.bin | --table\n"); return 2; }
    FILE* f = fopen(argv[1], "rb");
    FILE* g = fopen(argv[2], "wb");
    if (!f || !g) { printf("cannot open files\n"); return 2; }
    uint64_t blocks = 0;
    if (fread(&blocks, 8, 1, f) != 1) return 2;
    for (uint64_t b = 0; b < blocks; ++b) {
        uint64_t hdr[3];
        if (fread(hdr, 8, 3, f) != 3) { printf("short read\n"); return 2; }
        const int op = (int)hdr[0];
        const size_t n = hdr[1];
        int in_w, out_w;
        arith_words(op, &in_w, &out_w);
        if (in_w == 0 || (uint64_t)in_w != hdr[2]) { printf("op %d: record of %d words, file says %llu\n", op, in_w, (unsigned long long)hdr[2]); return 1; }
        std::vector<uint64_t> in(n * in_w), out(n * out_w, ~0ull);      // unwritten words stay all-ones
        if (fread(in.data(), 8, in.size(), f) != in.size()) { printf("short read\n"); return 2; }
        if (!run(op, in.data(), out.data(), n, in_w, out_w)) { printf("op %d has no host body\n", op); return 1; }
        if (fwrite(out.data(), 8, out.size(), g) != out.size()) return 2;
    }
    fclose(f);
    fclose(g);
    printf("ALL OK %llu\n", (unsigned long long)blocks);
    return 0;
}
