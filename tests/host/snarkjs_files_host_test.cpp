// csrc/snarkjs_files.h on the host, driven by tests/test_zkey_native_host.py.  Each argument after the mode is a file; the
// result for each is printed followed by a 0x1E record separator.
//   zkey <file>...    OK n_vars n_public domain_size n_coef n_bad first_bad   (records checked with coef_record_ok)  | ERR <message>
//   wtns <file>...    OK n                                                                                        | ERR <message>
//   proof <file>...   proof.json of 256 bytes: the fmt-0 encodings of A (64), C (64) and B (128)
//   public <file>...  public.json of the file's 32-byte little-endian values
#include <stdio.h>
#include <string.h>

#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "../../distributed_groth16_b200/csrc/snarkjs_files.h"

using namespace b200zk::sjf;

static std::vector<uint8_t> slurp(const char* path) {
    std::ifstream f(path, std::ios::binary);
    return std::vector<uint8_t>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const std::string mode = argv[1];
    for (int i = 2; i < argc; ++i) {
        const std::vector<uint8_t> b = slurp(argv[i]);
        const uint8_t* p = b.empty() ? (const uint8_t*)"" : b.data();
        std::string out, err;
        if (mode == "zkey") {
            Zkey z;
            if (!parse_zkey(p, b.size(), &z, &err)) {
                out = "ERR " + err;
            } else {
                unsigned long long bad = 0, first = z.n_coef;
                for (uint32_t k = 0; k < z.n_coef; ++k) {
                    const uint8_t* r = p + z.coef + 44ull * k;
                    if (!coef_record_ok(rd32(r), rd32(r + 4), rd32(r + 8), z.n_vars, z.domain_size)) {
                        if (!bad) first = k;
                        ++bad;
                    }
                }
                char s[160];
                snprintf(s, sizeof(s), "OK %u %u %u %u %llu %llu", z.n_vars, z.n_public, z.domain_size, z.n_coef, bad, first);
                out = s;
            }
        } else if (mode == "wtns") {
            Wtns w;
            out = parse_wtns(p, b.size(), &w, &err) ? "OK " + std::to_string(w.n) : "ERR " + err;
        } else if (mode == "proof") {
            if (b.size() != 256) return 3;
            out = proof_json(p, p + 128, p + 64);
        } else if (mode == "public") {
            out = public_json(p, b.size() / 32);
        } else {
            return 2;
        }
        fwrite(out.data(), 1, out.size(), stdout);
        fputc(0x1E, stdout);
    }
    return 0;
}
