// ORACLE — TEST INFRASTRUCTURE ONLY (see mj.h).
// Restates libriichi bin/validate_logs.rs:62-242 process_path over the oracle PlayerState: the checks of every event, then
// update(ev, keep_cans_on_announce = true) for seats 0..3; the first failure ends the log.
// Part of oracle/liboracle.so; tests/validate_lib.py binds the C entry points at the end of this file. orcv_init loads the tables
// for a library built from the oracle sources without capi.cc (in liboracle.so, orc_init has already loaded them).
#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "../include/mjx.h"
#include "state.h"

namespace orc {

struct Verdict { int32_t status = 0, reason = 0, line = 0, seat = -1; };  // include/mjx.h mjx_verdict

static Verdict check(int reason, int line, int actor) { Verdict v; v.status = MJX_V_CHECK; v.reason = reason; v.line = line; v.seat = actor; return v; }

// the error an update raised (state.cc ORC_ENSURE texts) -> a verdict reason
static int update_reason(const char* what) {
    const std::string m(what);
    if (m.find("exhausted yama") != std::string::npos) return MJX_R_EXHAUSTED_YAMA;
    if (m.find("unknown tile") != std::string::npos) return MJX_R_UNKNOWN_TILE;
    if (m.find("fifth") != std::string::npos) return MJX_R_FIFTH_TILE;
    if (m.find("discard from void") != std::string::npos) return MJX_R_DISCARD_FROM_VOID;
    if (m.find("consume from void") != std::string::npos) return MJX_R_CONSUME_FROM_VOID;
    if (m.find("too many dora indicators") != std::string::npos) return MJX_R_DORA_OVERFLOW;
    return MJX_R_UPDATE_OTHER;
}

// `ura_present[i]`: whether event i (a hora) carries `ura_markers` (Event keeps only the tiles)
static Verdict validate_log(const Event* evs, const bool* ura_present, int n) {
    PlayerState st[4] = {PlayerState(0), PlayerState(1), PlayerState(2), PlayerState(3)};
    ActionCandidate cans[4];
    for (int idx = 0; idx < n; idx++) {
        const Event& ev = evs[idx];
        const int line = idx + 1, a = ev.actor & 3;
        const ActionCandidate& c = cans[a];
        PlayerState& s = st[a];
        switch (ev.type) {
            case EV_DAHAI: {
                if (!c.can_discard) return check(MJX_R_CAN_DISCARD, line, a);
                bool dc[37];
                s.discard_candidates_aka(dc);
                if (ev.pai >= 37 || !dc[ev.pai]) return check(MJX_R_DISCARD_CANDIDATES, line, a);
                break;
            }
            case EV_CHI: {
                if ((ev.target + 1) % 4 != a) return check(MJX_R_CHI_NON_KAMICHA, line, a);
                const int x = deaka(ev.consumed[0]), y = deaka(ev.consumed[1]), t = deaka(ev.pai);  // chi_type.rs:12-25
                if (t < std::min(x, y)) { if (!c.can_chi_low) return check(MJX_R_CAN_CHI_LOW, line, a); }
                else if (t < std::max(x, y)) { if (!c.can_chi_mid) return check(MJX_R_CAN_CHI_MID, line, a); }
                else if (!c.can_chi_high) return check(MJX_R_CAN_CHI_HIGH, line, a);
                break;
            }
            case EV_PON: if (!c.can_pon) return check(MJX_R_CAN_PON, line, a); break;
            case EV_DAIMINKAN: if (!c.can_daiminkan) return check(MJX_R_CAN_DAIMINKAN, line, a); break;
            case EV_ANKAN: {
                if (!c.can_ankan) return check(MJX_R_CAN_ANKAN, line, a);
                const auto& v = s.ankan_candidates;
                if (std::find(v.begin(), v.end(), (u8)deaka(ev.consumed[0])) == v.end()) return check(MJX_R_ANKAN_CANDIDATES, line, a);
                break;
            }
            case EV_KAKAN: {
                if (!c.can_kakan) return check(MJX_R_CAN_KAKAN, line, a);
                const auto& v = s.kakan_candidates;
                if (std::find(v.begin(), v.end(), (u8)deaka(ev.pai)) == v.end()) return check(MJX_R_KAKAN_CANDIDATES, line, a);
                break;
            }
            case EV_REACH: if (!c.can_riichi) return check(MJX_R_CAN_RIICHI, line, a); break;
            case EV_HORA: {
                const bool is_ron = a != ev.target;
                if (is_ron && !c.can_ron_agari) return check(MJX_R_CAN_RON_AGARI, line, a);
                if (!is_ron && !c.can_tsumo_agari) return check(MJX_R_CAN_TSUMO_AGARI, line, a);
                // "This is a rough test / TODO: fix bug for double chankan ron" — kept as the reference has it
                if (!ura_present[idx]) return check(MJX_R_MISSING_URA, line, a);
                if (!ev.has_deltas) return check(MJX_R_MISSING_DELTAS, line, a);
                Point p;
                try { p = s.agari_points(is_ron, ev.ura_markers, ev.n_ura); }
                catch (const std::exception&) { return check(MJX_R_AGARI_POINTS, line, a); }
                const i32 need = is_ron ? p.ron : (s.is_oya() ? p.tsumo_oya : p.tsumo_ko);
                if (!(ev.deltas[a] >= need)) return check(MJX_R_DELTAS_BELOW_POINTS, line, a);
                break;
            }
            default: break;
        }
        for (int k = 0; k < 4; k++) {
            try {
                cans[k] = st[k].update(ev, /*keep_cans_on_announce=*/true);
            } catch (const OrcError& e) {
                Verdict v; v.status = MJX_V_UPDATE; v.reason = update_reason(e.what()); v.line = line; v.seat = k; return v;
            } catch (const std::exception&) {
                Verdict v; v.status = MJX_V_UPDATE; v.reason = MJX_R_UPDATE_OTHER; v.line = line; v.seat = k; return v;
            }
        }
    }
    return Verdict{};
}

}  // namespace orc

// ---------------- C ABI for ctypes ----------------
namespace {
thread_local std::string g_err;

// the flat event of the oracle's C ABI (oracle/capi.cc orc_event; tests/oracle_lib.py OrcEvent builds it from mjai JSON)
struct orcv_event {
    uint8_t type, actor, target, pai, tsumogiri;
    uint8_t consumed[4];
    uint8_t bakaze, kyoku, honba, kyotaku, oya;
    int32_t scores[4];
    uint8_t tehais[4][13];
    uint8_t has_deltas;  // bit 0: `deltas` present, bit 1: `ura_markers` present (a hora)
    int32_t deltas[4];
    uint8_t ura_markers[5];
    uint8_t n_ura;
};
static_assert(sizeof(orcv_event) == 112, "layout of oracle/capi.cc orc_event");
}  // namespace

extern "C" {

const char* orcv_last_error() { return g_err.c_str(); }

int orcv_init(const char* data_dir) {
    try { orc::tables_init(data_dir); return 0; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// process_path over one log: evs[n] in log order -> verdict4 = include/mjx.h mjx_verdict {status, reason, line, seat}
int orcv_validate_log(const orcv_event* evs, int n, int32_t* verdict4) {
    try {
        const size_t m = (size_t)std::max(n, 0);
        std::vector<orc::Event> e(m);
        std::unique_ptr<bool[]> ura(new bool[m + 1]);
        for (int i = 0; i < n; i++) {
            const orcv_event& c = evs[i];
            orc::Event& x = e[i];
            x.type = c.type; x.actor = c.actor; x.target = c.target; x.pai = c.pai; x.tsumogiri = c.tsumogiri != 0;
            memcpy(x.consumed, c.consumed, 4);
            x.bakaze = c.bakaze; x.kyoku = c.kyoku; x.honba = c.honba; x.kyotaku = c.kyotaku; x.oya = c.oya;
            memcpy(x.scores, c.scores, sizeof x.scores);
            memcpy(x.tehais, c.tehais, sizeof x.tehais);
            x.has_deltas = (c.has_deltas & 1) != 0;
            memcpy(x.deltas, c.deltas, sizeof x.deltas);
            memcpy(x.ura_markers, c.ura_markers, 5);
            x.n_ura = c.n_ura;
            ura[i] = (c.has_deltas & 2) != 0;
        }
        const orc::Verdict v = orc::validate_log(e.data(), ura.get(), n);
        verdict4[0] = v.status; verdict4[1] = v.reason; verdict4[2] = v.line; verdict4[3] = v.seat;
        return 0;
    } catch (const std::exception& ex) { g_err = ex.what(); return -1; }
}

}  // extern "C"
