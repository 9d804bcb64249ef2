// b200zk-prove [--device N | --devices I,J,...] <circuit.zkey> <witness.wtns> <proof.json> <public.json>
//
// snarkjs `groth16 prove` as one process, with the positional arguments of rapidsnark's prover: the zkey is loaded without
// fixed-base tables (table_window 0xFFFFFFFF: one proof does not pay back their build), r and s are drawn from the OS, and
// proof.json / public.json are written as snarkjs writes them.  --device N proves on one GPU (b200zk_zkey_*), --devices on a
// group of 1, 2, 4 or 8 of them (b200zk_group_zkey_*; an id may repeat, which emulates the group on fewer GPUs).  A usage
// error exits 2 before any CUDA call.  On any other failure it prints the library's message on stderr, exits 1 and leaves
// neither output file behind.
#include <errno.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <string>
#include <vector>

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

// "0,1,2,3" -> ids; false for an empty or malformed list or a count other than 1, 2, 4 or 8
bool parse_devices(const char* s, std::vector<int>* ids) {
    for (const char* p = s;; ++p) {
        char* end = nullptr;
        if (*p < '0' || *p > '9') return false;
        const long v = strtol(p, &end, 10);
        if (v > 1 << 20) return false;
        ids->push_back((int)v);
        p = end;
        if (*p == 0) break;
        if (*p != ',') return false;
    }
    const size_t n = ids->size();
    return n == 1 || n == 2 || n == 4 || n == 8;
}

// the two texts; on failure *err holds the library's message (context or group) or the failed create's code
struct Outputs {
    std::string proof_json, public_json;
};

int prove_one(int device, const Mapped& zkey, const Mapped& wtns, Outputs* out, std::string* err) {
    b200zk_ctx* ctx = nullptr;
    const int rc_ctx = b200zk_ctx_create(device, &ctx);
    if (rc_ctx != B200ZK_OK) {
        // no context, so no library message: the code says what kind of failure it was
        *err = "could not create a context on CUDA device " + std::to_string(device) + ": b200zk_ctx_create returned " +
               std::to_string(rc_ctx) + (rc_ctx == B200ZK_ERR_CUDA ? " (B200ZK_ERR_CUDA: the device is missing, or the CUDA "
                                                                     "runtime could not set it up)" : "");
        return rc_ctx;
    }
    b200zk_zkey* zk = nullptr;
    out->proof_json.assign(B200ZK_PROOF_JSON_MAX, '\0');
    int rc = b200zk_zkey_load(ctx, zkey.p == MAP_FAILED ? "" : zkey.p, zkey.len, 0xFFFFFFFFu, &zk);
    if (rc == B200ZK_OK) {
        size_t n_public = 0;
        b200zk_zkey_info(zk, nullptr, &n_public, nullptr, nullptr);
        out->public_json.assign(B200ZK_PUBLIC_JSON_MAX(n_public), '\0');
        size_t proof_len = out->proof_json.size(), public_len = out->public_json.size();
        const void* w = wtns.p == MAP_FAILED ? "" : wtns.p;
        rc = b200zk_zkey_prove(ctx, zk, w, wtns.len, nullptr, nullptr, nullptr, &out->proof_json[0], &proof_len, &out->public_json[0],
                               &public_len);
        if (rc == B200ZK_OK) {
            out->proof_json.resize(proof_len);
            out->public_json.resize(public_len);
        }
    }
    if (rc != B200ZK_OK) *err = b200zk_last_error(ctx);
    b200zk_zkey_free(ctx, zk);
    b200zk_ctx_destroy(ctx);
    return rc;
}

int prove_group(const std::vector<int>& ids, const Mapped& zkey, const Mapped& wtns, Outputs* out, std::string* err) {
    b200zk_group* grp = nullptr;
    const int rc_grp = b200zk_group_create(ids.data(), (int)ids.size(), &grp);
    if (rc_grp != B200ZK_OK) {
        // no group, so no library message
        *err = "could not create a group on the CUDA devices given: b200zk_group_create returned " + std::to_string(rc_grp) +
               (rc_grp == B200ZK_ERR_CUDA ? " (B200ZK_ERR_CUDA: a device is missing, two devices cannot reach each other, or the "
                                            "CUDA runtime could not set one up)" : "");
        return rc_grp;
    }
    b200zk_group_zkey* zk = nullptr;
    out->proof_json.assign(B200ZK_PROOF_JSON_MAX, '\0');
    int rc = b200zk_group_zkey_load(grp, zkey.p == MAP_FAILED ? "" : zkey.p, zkey.len, 0xFFFFFFFFu, &zk);
    if (rc == B200ZK_OK) {
        size_t n_public = 0;
        b200zk_group_zkey_info(zk, nullptr, &n_public, nullptr, nullptr);
        out->public_json.assign(B200ZK_PUBLIC_JSON_MAX(n_public), '\0');
        size_t proof_len = out->proof_json.size(), public_len = out->public_json.size();
        const void* w = wtns.p == MAP_FAILED ? "" : wtns.p;
        rc = b200zk_group_zkey_prove(grp, zk, w, wtns.len, nullptr, nullptr, nullptr, &out->proof_json[0], &proof_len,
                                     &out->public_json[0], &public_len);
        if (rc == B200ZK_OK) {
            out->proof_json.resize(proof_len);
            out->public_json.resize(public_len);
        }
    }
    if (rc != B200ZK_OK) *err = b200zk_group_last_error(grp);
    b200zk_group_zkey_free(grp, zk);
    b200zk_group_destroy(grp);
    return rc;
}

}  // namespace

int main(int argc, char** argv) {
    int device = 0, a = 1;
    std::vector<int> ids;
    bool usage = false;
    if (argc == 7 && strcmp(argv[1], "--device") == 0) {
        char* end = nullptr;
        device = (int)strtol(argv[2], &end, 10);
        usage = !*argv[2] || *end;
        a = 3;
    } else if (argc == 7 && strcmp(argv[1], "--devices") == 0) {
        usage = !parse_devices(argv[2], &ids);
        a = 3;
    }
    if (usage || argc - a != 4) {
        fprintf(stderr, "usage: b200zk-prove [--device N | --devices I,J,... (1, 2, 4 or 8 ids)] <circuit.zkey> <witness.wtns> "
                        "<proof.json> <public.json>\n");
        return 2;
    }
    const char *zkey_path = argv[a], *wtns_path = argv[a + 1];
    const std::string proof_path = argv[a + 2], public_path = argv[a + 3];
    std::string err;
    Mapped zkey, wtns;
    if (!map_file(zkey_path, &zkey, &err) || !map_file(wtns_path, &wtns, &err)) return fail(err);

    Outputs out;
    const int rc = ids.empty() ? prove_one(device, zkey, wtns, &out, &err) : prove_group(ids, zkey, wtns, &out, &err);
    if (rc != B200ZK_OK) return fail(err);

    const std::string proof_tmp = proof_path + ".tmp", public_tmp = public_path + ".tmp";
    if (!write_tmp(proof_tmp, out.proof_json.data(), out.proof_json.size(), &err)) return fail(err);
    if (!write_tmp(public_tmp, out.public_json.data(), out.public_json.size(), &err)) {
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
