// TEST INFRASTRUCTURE ONLY — host build of the training-buffer observation codec (mortal_b200/csrc/mjx_obs_pack.cuh, the record
// layout of csrc/mjx_obs.cuh make_obs_record, -DMJX_HOST_EMUL): k_obs_pack's work one sample at a time and k_obs_unpack's through
// the host enc_materialize, slice by slice, so the codec can be checked on oracle observations and run under sanitizers without a
// GPU. Never loaded by mortal_b200/. Part of libmjx_emul.so (tests/emul_lib.py); bound by tests/obs_pack_lib.py.
#include <cstdint>
#include <cstring>

#include "mjx_obs_pack.cuh"

using namespace mjx;

extern "C" {

int emulp_record_bytes(int version, int invisible) {
    if (version < 1 || version > 4 || (invisible != 0 && invisible != 1)) return -2;
    return make_obs_record(version, invisible != 0).bytes;
}

// mjx_obs_pack_dev over host arrays: the same argument checks (returns -2 where they fail)
int emulp_pack(int version, int invisible, long long n, const float* obs, long long sample_pitch, uint8_t* records, int32_t* status) {
    if (obs_pack_check(version, invisible, n, obs, sample_pitch, records, status)) return -2;
    const ObsRecord R = make_obs_record(version, invisible != 0);
    const ObsPackSlices P = make_pack_slices(R);
    for (long long i = 0; i < n; i++) status[i] = obs_pack_sample(R, P, obs + i * sample_pitch, records + i * R.bytes);
    return 0;
}

// mjx_obs_unpack_dev over host arrays
int emulp_unpack(int version, int invisible, const uint8_t* records, long long n_records, const int64_t* idx, long long n_idx,
                 float* out) {
    if (obs_unpack_check(version, invisible, records, n_records, idx, n_idx, out)) return -2;
    const ObsRecord R = make_obs_record(version, invisible != 0);
    static const uint64_t zero[(OBS_ROWS_V4 * 8 + OBS_REC_MAX_VAL * OBS_COLS * 4) / 8] = {};
    for (long long b = 0; b < n_idx; b++) {
        const long long k = idx[b];
        const uint8_t* rec = k >= 0 && k < n_records ? records + k * R.bytes : reinterpret_cast<const uint8_t*>(zero);
        float* dst = out + b * R.rows * OBS_COLS;
        for (int lo = 0; lo < R.rows; lo += OBS_SLICE_ROWS)
            enc_materialize(reinterpret_cast<const u64*>(rec), R.rows, reinterpret_cast<const float*>(rec + R.rows * 8), R.val_row,
                            R.n_val, dst + lo * OBS_COLS, lo, lo + OBS_SLICE_ROWS < R.rows ? lo + OBS_SLICE_ROWS : R.rows);
    }
    return 0;
}

// the record layout: value rows of (version, invisible) into val_rows (OBS_REC_MAX_VAL shorts); returns their count
int emulp_value_rows(int version, int invisible, int16_t* val_rows) {
    if (version < 1 || version > 4 || (invisible != 0 && invisible != 1)) return -2;
    const ObsRecord R = make_obs_record(version, invisible != 0);
    for (int k = 0; k < R.n_val; k++) val_rows[k] = R.val_row[k];
    return R.n_val;
}

}  // extern "C"
