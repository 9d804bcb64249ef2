// b200zk-prove [--device N] <circuit.zkey> <witness.wtns> <proof.json> <public.json>
//
// snarkjs `groth16 prove` as one process, with the positional arguments of rapidsnark's prover: the zkey is loaded without
// fixed-base tables (b200zk_zkey_load, table_window 0xFFFFFFFF: one proof does not pay back their build), r and s are drawn
// from the OS, and proof.json / public.json are written as snarkjs writes them.  On any failure it prints the library's
// message on stderr, exits non-zero and leaves neither output file behind.
#include <errno.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <string>

#include "../../include/b200zk.h"

namespace {

struct Mapped {
    void* p = MAP_FAILED;
    size_t len = 0;
    ~Mapped() { if (p != MAP_FAILED && len) munmap(p, len); }
};

bool map_file(const char* path, Mapped* m, std::string* err) {
    const int fd = open(path, O_RDONLY);
    if (fd < 0) { *err = std::string(path) + ": " + strerror(errno); return false; }
    struct stat st;
    if (fstat(fd, &st) != 0) { *err = std::string(path) + ": " + strerror(errno); close(fd); return false; }
    m->len = (size_t)st.st_size;
    if (m->len) {
        m->p = mmap(nullptr, m->len, PROT_READ, MAP_PRIVATE, fd, 0);
        if (m->p == MAP_FAILED) { *err = std::string(path) + ": " + strerror(errno); close(fd); return false; }
    }
    close(fd);
    return true;
}

// the whole text into path.tmp, renamed by the caller once both files are complete
bool write_tmp(const std::string& path, const char* text, size_t len, std::string* err) {
    FILE* f = fopen(path.c_str(), "wb");
    if (!f) { *err = path + ": " + strerror(errno); return false; }
    const bool ok = fwrite(text, 1, len, f) == len;
    if (fclose(f) != 0 || !ok) { *err = path + ": write failed"; unlink(path.c_str()); return false; }
    return true;
}

int fail(const std::string& msg) {
    fprintf(stderr, "b200zk-prove: %s\n", msg.c_str());
    return 1;
}

}  // namespace

int main(int argc, char** argv) {
    int device = 0, a = 1;
    if (argc == 7 && strcmp(argv[1], "--device") == 0) {
        char* end = nullptr;
        device = (int)strtol(argv[2], &end, 10);
        if (!*argv[2] || *end) argc = 0;
        a = 3;
    }
    if (argc - a != 4) {
        fprintf(stderr, "usage: b200zk-prove [--device N] <circuit.zkey> <witness.wtns> <proof.json> <public.json>\n");
        return 2;
    }
    const char *zkey_path = argv[a], *wtns_path = argv[a + 1];
    const std::string proof_path = argv[a + 2], public_path = argv[a + 3];
    std::string err;
    Mapped zkey, wtns;
    if (!map_file(zkey_path, &zkey, &err) || !map_file(wtns_path, &wtns, &err)) return fail(err);

    b200zk_ctx* ctx = nullptr;
    const int rc_ctx = b200zk_ctx_create(device, &ctx);
    if (rc_ctx != B200ZK_OK) {
        // no context, so no library message: the code says what kind of failure it was
        return fail("could not create a context on CUDA device " + std::to_string(device) + ": b200zk_ctx_create returned " +
                    std::to_string(rc_ctx) + (rc_ctx == B200ZK_ERR_CUDA ? " (B200ZK_ERR_CUDA: the device is missing, or the CUDA "
                                                                          "runtime could not set it up)" : ""));
    }
    b200zk_zkey* zk = nullptr;
    std::string proof_json(B200ZK_PROOF_JSON_MAX, '\0'), public_json;
    int rc = b200zk_zkey_load(ctx, zkey.p == MAP_FAILED ? "" : zkey.p, zkey.len, 0xFFFFFFFFu, &zk);
    if (rc == B200ZK_OK) {
        size_t n_public = 0;
        b200zk_zkey_info(zk, nullptr, &n_public, nullptr, nullptr);
        public_json.assign(B200ZK_PUBLIC_JSON_MAX(n_public), '\0');
        size_t proof_len = proof_json.size(), public_len = public_json.size();
        const void* w = wtns.p == MAP_FAILED ? "" : wtns.p;
        rc = b200zk_zkey_prove(ctx, zk, w, wtns.len, nullptr, nullptr, nullptr, &proof_json[0], &proof_len, &public_json[0], &public_len);
        if (rc == B200ZK_OK) {
            proof_json.resize(proof_len);
            public_json.resize(public_len);
        }
    }
    if (rc != B200ZK_OK) {
        err = b200zk_last_error(ctx);
        b200zk_zkey_free(ctx, zk);
        b200zk_ctx_destroy(ctx);
        return fail(err);
    }
    b200zk_zkey_free(ctx, zk);
    b200zk_ctx_destroy(ctx);

    const std::string proof_tmp = proof_path + ".tmp", public_tmp = public_path + ".tmp";
    if (!write_tmp(proof_tmp, proof_json.data(), proof_json.size(), &err)) return fail(err);
    if (!write_tmp(public_tmp, public_json.data(), public_json.size(), &err)) {
        unlink(proof_tmp.c_str());
        return fail(err);
    }
    if (rename(proof_tmp.c_str(), proof_path.c_str()) != 0) {
        err = proof_path + ": " + strerror(errno);
        unlink(proof_tmp.c_str());
        unlink(public_tmp.c_str());
        return fail(err);
    }
    if (rename(public_tmp.c_str(), public_path.c_str()) != 0) {
        err = public_path + ": " + strerror(errno);
        unlink(proof_path.c_str());
        unlink(public_tmp.c_str());
        return fail(err);
    }
    return 0;
}
