/* mjx_logio — reading log files on the device for libmjx.so's log decoder (csrc/mjx_inflate.cuh): gzip members inflated straight
 * into the text buffer mjx_mjai_count_dev reads, and a key count over that text. Same conventions as include/mjx.h: device
 * pointers, 0 or a negative mjx_status, `stream` a cudaStream_t passed as void*, enqueued without a synchronise.
 *
 * mjx_gunzip_dev: file i is gz[gz_off[i], gz_off[i + 1]), one gzip member (RFC 1952) whose deflate stream (RFC 1951) is inflated
 * into out[out_off[i], out_off[i + 1]) (gz_off, out_off int64 [n + 1]; the caller sizes each slot from the file's ISIZE, its last
 * four bytes). status int32 [n] gets one mjx_gunzip_status per file. OK means exactly: Python's gzip.decompress of the same bytes
 * succeeds and returns the bytes written to the slot, which fill it. Any other status declines the file: its slot's contents are
 * then unspecified and the caller reads the file on the host. Nothing is written at or past out_off[i + 1]. One warp per file. */
#ifndef MJX_LOGIO_H
#define MJX_LOGIO_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* The per-file status: X(enum suffix, name). This list is the single definition (mortal_b200/_logio.py reads it).
 *   NOT_GZIP   no gzip magic (1f 8b) or a compression method other than 8
 *   HEADER     the header's optional fields (FEXTRA, FNAME, FCOMMENT, FHCRC) run past the file
 *   BLOCK      block type 3, or a stored block whose LEN and NLEN do not match
 *   CODES      HLIT > 286, HDIST > 30, an over-subscribed or incomplete code (a distance code may be empty or a single length-1
 *              code), a repeat code with nothing to repeat or running past the count, no end-of-block code
 *   SYMBOL     length symbol 286 / 287, distance symbol 30 / 31, a bit pattern no code has
 *   DISTANCE   a distance back past the start of the output
 *   TRUNCATED  the deflate stream or its 8-byte trailer runs past the file
 *   SIZE       output other than ISIZE, or past the slot
 *   CRC        the output's CRC-32 differs from the trailer's
 *   TRAILING   any byte after the member's trailer (zero padding, a second member, garbage) */
#define MJX_GUNZIP_STATUSES(X)                                                                                               \
    X(OK, "ok") X(NOT_GZIP, "not_gzip") X(HEADER, "header") X(BLOCK, "block") X(CODES, "codes") X(SYMBOL, "symbol")         \
    X(DISTANCE, "distance") X(TRUNCATED, "truncated") X(SIZE, "size") X(CRC, "crc") X(TRAILING, "trailing")
#define MJX_GUNZIP_ENUM_(id, name) MJX_GZ_##id,
enum mjx_gunzip_status { MJX_GUNZIP_STATUSES(MJX_GUNZIP_ENUM_) MJX_GZ_COUNT };
#undef MJX_GUNZIP_ENUM_

int mjx_gunzip_dev(int n, const uint8_t* gz, long long n_gz, const int64_t* gz_off, uint8_t* out, long long n_out,
                   const int64_t* out_off, int32_t* status, void* stream);

/* Python's bytes.count of every key over every log's text: counts int64 [n_logs, n_keys], occurrences counted left to right
 * without overlap. text / log_off as in mjx_mjai_count_dev (device); the keys are host memory, key k = keys_host[key_off_host[k],
 * key_off_host[k + 1]) with 1 <= n_keys <= MJX_COUNT_KEYS_MAX and every key 1..MJX_COUNT_KEY_BYTES bytes long. */
#define MJX_COUNT_KEYS_MAX 8
#define MJX_COUNT_KEY_BYTES 16
int mjx_count_keys_dev(int n_logs, const uint8_t* text, long long n_bytes, const int64_t* log_off, const uint8_t* keys_host,
                       const int32_t* key_off_host, int n_keys, int64_t* counts, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MJX_LOGIO_H */
