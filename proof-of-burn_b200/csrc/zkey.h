// zkey.h -- the section table of a snarkjs Groth16 `.zkey` (format: include/pob_b200.h, DESIGN.md §5 "Key loading"), parsed and
// validated on the host by zkey.cpp; pob_zkey_load (pob_b200.cu) streams the sections it locates.
#pragma once
#include <stdint.h>
#include <stdexcept>
#include <string>
#include "../../include/pob_b200.h"

namespace pob {

enum { ZK_N_IDS = 10, ZK_SEC2_BYTES = 660, ZK_SEC2_POINTS = 84, ZK_ENTRY_BYTES = 44 };

struct ZkeyLayout {
    uint64_t off[ZK_N_IDS] = {}, size[ZK_N_IDS] = {};    // content offset and size of sections 1..9 (index = id)
    uint64_t n_vars = 0, n_coefs = 0, domain = 0, file_bytes = 0;
    uint32_t n_pub = 0, log_n = 0;
    uint8_t sec2[ZK_SEC2_BYTES] = {};                      // section 2 as read
    pob_zkey_desc desc{};
};

// thrown by zkey_parse: code is POB_E_IO or POB_E_KEY
struct ZkeyError : std::runtime_error {
    int code;
    ZkeyError(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

ZkeyLayout zkey_parse(const char *path);
// read exactly `bytes` at `off` (false on a read error or end of file)
bool zkey_pread(int fd, void *dst, uint64_t bytes, uint64_t off);

}  // namespace pob
