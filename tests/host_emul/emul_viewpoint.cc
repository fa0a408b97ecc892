// TEST INFRASTRUCTURE ONLY — the single-lane host build of tests/host_emul/emul.cc plus the scan of k_replay_viewpoints
// (csrc/mjx_replay.cuh replay_hidden_seats / replay_mark_viewpoint), so single-viewpoint replays can be diffed against the oracle
// and run under sanitizers without a GPU. Never loaded by mortal_b200/. Built by tests/viewpoint_lib.py.
#include "emul.cc"

extern "C" {

// mjx_env_replay_viewpoints on an emul_replay_create env: the scan and the mark, one lane per job; the scan result of every job
// (-1 = not marked, else the mask of hidden seats) goes to `masks` when it is not null
void emul_replay_viewpoints(void* p, int32_t* masks) {
    EmulEnv* E = static_cast<EmulEnv*>(p);
    const long long n_hdr = (long long)E->r_hdr.size(), n_kyoku = (long long)(E->r_kyoku.size() / REPLAY_KYOKU_WORDS);
    for (int t = 0; t < E->n; t++) {
        const int mask = replay_hidden_seats(E->R, t, n_hdr, n_kyoku, 0);
        replay_mark_viewpoint(&E->tabs[t], E->R.player[t], mask);
        if (masks) masks[t] = mask;
    }
}

}  // extern "C"
