// zkey.cpp -- host-side reading of a snarkjs `.zkey` header and section table (pob_zkey_info), no GPU needed.  Only the header,
// the section table, section 2 and the first word of section 4 are read; pob_zkey_load streams the rest.
#include "zkey.h"
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <algorithm>
#include <cstring>

namespace pob {

// BN254's base field q and scalar field r, 32-byte little endian
static const uint8_t ZK_Q[32] = {0x47, 0xfd, 0x7c, 0xd8, 0x16, 0x8c, 0x20, 0x3c, 0x8d, 0xca, 0x71, 0x68, 0x91, 0x6a, 0x81, 0x97,
                                 0x5d, 0x58, 0x81, 0x81, 0xb6, 0x45, 0x50, 0xb8, 0x29, 0xa0, 0x31, 0xe1, 0x72, 0x4e, 0x64, 0x30};
static const uint8_t ZK_R[32] = {0x01, 0x00, 0x00, 0xf0, 0x93, 0xf5, 0xe1, 0x43, 0x91, 0x70, 0xb9, 0x79, 0x48, 0xe8, 0x33, 0x28,
                                 0x5d, 0x58, 0x81, 0x81, 0xb6, 0x45, 0x50, 0xb8, 0x29, 0xa0, 0x31, 0xe1, 0x72, 0x4e, 0x64, 0x30};

bool zkey_pread(int fd, void *dst, uint64_t bytes, uint64_t off) {
    uint8_t *p = (uint8_t *)dst;
    while (bytes) {
        const ssize_t r = pread(fd, p, (size_t)std::min<uint64_t>(bytes, 1ull << 30), (off_t)off);
        if (r <= 0) return false;
        p += r; bytes -= (uint64_t)r; off += (uint64_t)r;
    }
    return true;
}

namespace {
struct Fd {
    int fd;
    explicit Fd(int f) : fd(f) {}
    ~Fd() { if (fd >= 0) close(fd); }
};
uint32_t u32_at(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
[[noreturn]] void key_error(const std::string &m) { throw ZkeyError(POB_E_KEY, m); }
}  // namespace

ZkeyLayout zkey_parse(const char *path) {
    ZkeyLayout L;
    Fd f(open(path, O_RDONLY));
    if (f.fd < 0) throw ZkeyError(POB_E_IO, std::string("cannot open ") + path);
    struct stat st;
    if (fstat(f.fd, &st) != 0) throw ZkeyError(POB_E_IO, std::string("cannot stat ") + path);
    L.file_bytes = (uint64_t)st.st_size;
    auto rd = [&](void *dst, uint64_t bytes, uint64_t off, const std::string &what) {
        if (off > L.file_bytes || bytes > L.file_bytes - off) throw ZkeyError(POB_E_IO, "the file ends early, inside " + what);
        if (!zkey_pread(f.fd, dst, bytes, off)) throw ZkeyError(POB_E_IO, "read error in " + what);
    };
    uint8_t hd[12];
    rd(hd, 4, 0, "the magic");
    if (memcmp(hd, "zkey", 4) != 0) key_error("bad magic (not a .zkey file)");
    rd(hd + 4, 8, 4, "the header");
    if (u32_at(hd + 4) != 1) key_error("unsupported version " + std::to_string(u32_at(hd + 4)) + " (expected 1)");
    const uint32_t nsec = u32_at(hd + 8);
    uint64_t pos = 12;
    for (uint32_t k = 0; k < nsec; k++) {
        uint8_t sh[12];
        rd(sh, 12, pos, "the header of section entry " + std::to_string(k));
        const uint32_t id = u32_at(sh);
        uint64_t size; memcpy(&size, sh + 4, 8);
        pos += 12;
        if (pos > L.file_bytes || size > L.file_bytes - pos) throw ZkeyError(POB_E_IO, "the file ends early, inside section " + std::to_string(id));
        if (id >= 1 && id <= 9) {
            if (L.off[id]) key_error("section " + std::to_string(id) + " appears twice");
            L.off[id] = pos; L.size[id] = size;
        }
        pos += size;
    }
    if (pos != L.file_bytes) key_error("the file has " + std::to_string(L.file_bytes - pos) + " bytes after its last section");
    for (int id = 1; id <= 9; id++) if (!L.off[id]) key_error("section " + std::to_string(id) + " is missing");
    auto want = [&](int id, uint64_t bytes, const std::string &why) {
        if (L.size[id] != bytes) key_error("section " + std::to_string(id) + " has " + std::to_string(L.size[id]) + " bytes, " + why + " gives " + std::to_string(bytes));
    };
    want(1, 4, "the protocol word");
    uint8_t w[4];
    rd(w, 4, L.off[1], "section 1");
    if (u32_at(w) != 1) key_error("protocol " + std::to_string(u32_at(w)) + " is not Groth16 (1)");
    want(2, ZK_SEC2_BYTES, "the Groth16 header");
    rd(L.sec2, ZK_SEC2_BYTES, L.off[2], "section 2");
    const uint8_t *s2 = L.sec2;
    if (u32_at(s2) != 32) key_error("n8q is " + std::to_string(u32_at(s2)) + ", not 32");
    if (memcmp(s2 + 4, ZK_Q, 32) != 0) key_error("q is not BN254's base field modulus");
    if (u32_at(s2 + 36) != 32) key_error("n8r is " + std::to_string(u32_at(s2 + 36)) + ", not 32");
    if (memcmp(s2 + 40, ZK_R, 32) != 0) key_error("r is not BN254's scalar field modulus");
    L.n_vars = u32_at(s2 + 72); L.n_pub = u32_at(s2 + 76); L.domain = u32_at(s2 + 80);
    if (L.domain == 0 || (L.domain & (L.domain - 1)) || L.domain > (1ull << 28)) key_error("domainSize " + std::to_string(L.domain) + " is not a power of two <= 2^28");
    while ((1ull << L.log_n) < L.domain) L.log_n++;
    if (L.n_vars < (uint64_t)L.n_pub + 1) key_error("nVars " + std::to_string(L.n_vars) + " < nPublic + 1");
    want(3, 64ull * (L.n_pub + 1), "nPublic + 1 G1 points");
    if (L.size[4] < 4) key_error("section 4 has no coefficient count");
    rd(w, 4, L.off[4], "section 4");
    L.n_coefs = u32_at(w);
    want(4, 4 + (uint64_t)ZK_ENTRY_BYTES * L.n_coefs, "nCoefs");
    want(5, 64 * L.n_vars, "nVars G1 points");
    want(6, 64 * L.n_vars, "nVars G1 points");
    want(7, 128 * L.n_vars, "nVars G2 points");
    want(8, 64 * (L.n_vars - L.n_pub - 1), "nVars - nPublic - 1 G1 points");
    want(9, 64 * L.domain, "domainSize G1 points");
    pob_zkey_desc &d = L.desc;
    d.n_vars = L.n_vars; d.n_pub = L.n_pub; d.log_n = L.log_n; d.n_coefs = L.n_coefs; d.file_bytes = L.file_bytes;
    d.a_bytes = L.size[5]; d.b1_bytes = L.size[6]; d.b2_bytes = L.size[7]; d.c_bytes = L.size[8]; d.h_bytes = L.size[9];
    d.key_bytes = d.a_bytes + d.b1_bytes + d.b2_bytes + d.c_bytes + d.h_bytes + 3 * 64 + 2 * 128;
    return L;
}

}  // namespace pob

extern "C" int pob_zkey_info(const char *path, pob_zkey_desc *out);
// pob_last_error's message store lives in pob_b200.cu
void pob_set_error(const std::string &msg);

int pob_zkey_info(const char *path, pob_zkey_desc *out) {
    if (!path || !out) { pob_set_error("pob_zkey_info: null argument"); return POB_E_BAD_ARG; }
    try { *out = pob::zkey_parse(path).desc; }
    catch (const pob::ZkeyError &e) { pob_set_error(std::string("pob_zkey_info: ") + path + ": " + e.what()); return e.code; }
    return POB_OK;
}

extern "C" int pob_zkey_vk(const char *path, void *out, uint64_t out_bytes, uint32_t *n_pub);

int pob_zkey_vk(const char *path, void *out, uint64_t out_bytes, uint32_t *n_pub) {
    if (!path || !out || !n_pub) { pob_set_error("pob_zkey_vk: null argument"); return POB_E_BAD_ARG; }
    try {
        const pob::ZkeyLayout L = pob::zkey_parse(path);
        *n_pub = L.n_pub;
        const uint64_t need = 448 + L.size[3];
        if (out_bytes < need) { pob_set_error("pob_zkey_vk: out holds " + std::to_string(out_bytes) + " bytes, the key has " + std::to_string(need)); return POB_E_BAD_ARG; }
        uint8_t *o = (uint8_t *)out;
        const uint8_t *s2 = L.sec2 + 84;                                   // alpha1, beta1, beta2, gamma2, delta1, delta2
        memcpy(o, s2, 64);                                                 // alpha1
        memcpy(o + 64, s2 + 128, 256);                                     // beta2, gamma2
        memcpy(o + 320, s2 + 448, 128);                                    // delta2
        pob::Fd f(open(path, O_RDONLY));
        if (f.fd < 0 || !pob::zkey_pread(f.fd, o + 448, L.size[3], L.off[3])) { pob_set_error(std::string("pob_zkey_vk: ") + path + ": read error in section 3"); return POB_E_IO; }
    } catch (const pob::ZkeyError &e) { pob_set_error(std::string("pob_zkey_vk: ") + path + ": " + e.what()); return e.code; }
    return POB_OK;
}
