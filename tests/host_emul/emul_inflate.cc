// TEST INFRASTRUCTURE ONLY — host build of mortal_b200/csrc/mjx_inflate.cuh (-DMJX_HOST_EMUL): k_gunzip's member decode and
// k_count_keys's window walk, one lane playing all 32 in turn (the table fills, the match and stored copies, the per-lane CRC
// chunks and their combination), so the accept / decline rule and the bytes can be diffed against Python's gzip and zlib and run
// under sanitizers without a GPU. Never loaded by mortal_b200/. Part of libmjx_emul.so (tests/emul_lib.py).
#include <cstdint>
#include <cstring>

#include "mjx_inflate.cuh"

using namespace mjx;

namespace {
struct CrcTables {
    u32 table[256], x8[GZ_X8];
    CrcTables() {
        for (u32 k = 0; k < 256; k++) table[k] = gz_crc_entry(k);
        gz_x8_table(x8);
    }
};
const CrcTables& crc_tables() {
    static const CrcTables T;
    return T;
}
}  // namespace

extern "C" {

// mjx_gunzip_dev over host arrays: the same arguments and per-file statuses. Returns 0 or -2.
int emulz_gunzip(int n, const uint8_t* gz, long long n_gz, const int64_t* gz_off, uint8_t* out, long long n_out,
                 const int64_t* out_off, int32_t* status) {
    if (n <= 0 || n_gz < 0 || !gz_off || !out_off || !status) return -2;
    const CrcTables& T = crc_tables();
    for (int i = 0; i < n; i++) {
        GzWarp W;  // uninitialised, as shared memory is
        const long long gb = gz_off[i], ge = gz_off[i + 1], ob = out_off[i], oe = out_off[i + 1];
        if (ob < 0 || oe < ob || oe > n_out) status[i] = MJX_GZ_SIZE;
        else if (gb < 0 || ge < gb || ge > n_gz) status[i] = MJX_GZ_NOT_GZIP;
        else status[i] = gz_member(W, gz, n_gz, gb, ge, out + ob, oe - ob, T.table, T.x8, 0);
    }
    return 0;
}

// zlib.crc32 of data[0, n) by the kernel's 32 lane chunks and their combination
uint32_t emulz_crc32(const uint8_t* data, long long n) {
    const CrcTables& T = crc_tables();
    return gz_crc32(data, n, T.table, T.x8, 0);
}

// mjx_count_keys_dev over host arrays. Returns 0 or -2.
int emulz_count_keys(int n_logs, const uint8_t* text, long long n_bytes, const int64_t* log_off, const uint8_t* keys,
                     const int32_t* key_off, int n_keys, int64_t* counts) {
    if (n_logs <= 0 || !log_off || n_keys < 1 || n_keys > MJX_COUNT_KEYS_MAX) return -2;
    GzKeys K{};
    K.n = n_keys;
    for (int k = 0; k < n_keys; k++) {
        K.len[k] = key_off[k + 1] - key_off[k];
        if (K.len[k] < 1 || K.len[k] > MJX_COUNT_KEY_BYTES) return -2;
        std::memcpy(K.b[k], keys + key_off[k], K.len[k]);
    }
    for (int i = 0; i < n_logs; i++) {
        long long lb = log_off[i], le = log_off[i + 1];
        if (lb < 0 || le < lb || le > n_bytes) lb = le = 0;
        long long cnt[MJX_COUNT_KEYS_MAX];
        gz_count_keys(text + lb, le - lb, K, cnt, 0);
        for (int k = 0; k < n_keys; k++) counts[(long long)i * n_keys + k] = cnt[k];
    }
    return 0;
}

}  // extern "C"
