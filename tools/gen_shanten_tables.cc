// Generates the two shanten lookup tables from first principles (no input files):
//   shanten_suhai.bin  5^9 = 1,953,125 rows  (index = base-5 number of the nine rank counts, rank 1 most significant)
//   shanten_jihai.bin  5^7 =    78,125 rows  (seven honour counts)
// Row = 10 nibbles: [m] for m = 0..4 is the minimum number of tiles that must still be ADDED to the suit so that it
// contains m complete melds, [5 + m] the same for m melds plus a pair; a target shape never uses more than four copies
// of a tile. These are the "distance" tables of the table-based shanten algorithm libriichi uses (algo/shanten.rs:27-84,
// 88-100: the per-suit rows are combined by a min-plus merge and 1 is subtracted at the end).
// Output format = the reference's unpacked table: 5 bytes per row, low nibble first (shanten.rs:27-44).
// tools/build_tables.py runs this and cross-checks the result byte for byte against the reference's own data files,
// stored in tests/golden/tables/ (tests/test_tables.py).
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

namespace {
constexpr int INF = 99;

// DP state after processing rank i: a = runs started at i-1 (need their third tile at i+1), b = runs started at i
// (need tiles at i+1 and i+2), m = melds so far, p = pair used. cost[a][b][m][p].
struct State { int8_t c[5][5][5][2]; };

void init(State& s) {
    memset(&s, INF, sizeof s);
    s.c[0][0][0][0] = 0;
}

// advance by one rank holding `have` tiles; `can_start_run` is false for ranks 8, 9 and for honours
void step(const State& f, State& g, int have, bool can_start_run) {
    memset(&g, INF, sizeof g);
    for (int a = 0; a < 5; a++)
        for (int b = 0; a + b < 5; b++)
            for (int m = 0; m < 5; m++)
                for (int p = 0; p < 2; p++) {
                    const int base = f.c[a][b][m][p];
                    if (base >= INF) continue;
                    const int cmax = can_start_run ? 4 - a - b : 0;
                    for (int c = 0; c <= cmax; c++)
                        for (int k = 0; k < 2; k++)
                            for (int q = 0; q + p < 2; q++) {
                                const int need = a + b + c + 3 * k + 2 * q;
                                const int m2 = m + c + k;
                                if (need > 4 || m2 > 4) continue;
                                const int cost = base + std::max(need - have, 0);
                                int8_t& dst = g.c[b][c][m2][p + q];
                                if (cost < dst) dst = (int8_t)cost;
                            }
                }
}

void emit(const State& f, std::vector<uint8_t>& out, size_t row) {
    int v[10];
    for (int m = 0; m < 5; m++) { v[m] = f.c[0][0][m][0]; v[5 + m] = f.c[0][0][m][1]; }
    for (int i = 0; i < 5; i++) out[row * 5 + i] = (uint8_t)((v[2 * i] & 15) | ((v[2 * i + 1] & 15) << 4));
}

void rec(const State& f, int depth, int n, size_t index, bool suhai, std::vector<uint8_t>& out) {
    if (depth == n) { emit(f, out, index); return; }
    for (int have = 0; have < 5; have++) {
        State g;
        step(f, g, have, suhai && depth < 7);
        rec(g, depth + 1, n, index * 5 + have, suhai, out);
    }
}

bool write_file(const char* path, const std::vector<uint8_t>& data) {
    FILE* fp = fopen(path, "wb");
    if (!fp) return false;
    const bool ok = fwrite(data.data(), 1, data.size(), fp) == data.size();
    fclose(fp);
    return ok;
}
}  // namespace

int main(int argc, char** argv) {
    if (argc != 3) { fprintf(stderr, "usage: %s <shanten_suhai.bin> <shanten_jihai.bin>\n", argv[0]); return 2; }
    State f;
    {
        std::vector<uint8_t> out((size_t)1953125 * 5);
        init(f);
        rec(f, 0, 9, 0, true, out);
        if (!write_file(argv[1], out)) return 1;
    }
    {
        std::vector<uint8_t> out((size_t)78125 * 5);
        init(f);
        rec(f, 0, 7, 0, false, out);
        if (!write_file(argv[2], out)) return 1;
    }
    return 0;
}
