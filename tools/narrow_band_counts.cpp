// narrow_band_counts.cpp -- the host build of the aligner (tests/hostsim/hostsim.cpp) with the scalar affine-gap form's counting
// points defined: for every banded call of up to 4 vectors per segment (the calls the second pass gives to the narrow-band forms),
// its (row, segment) units and the lazy-F rounds each entered.  From them, per call, what each narrow-band form runs:
//   rows (sg_warp_ag_rows_banded4): one warp step per unit, the unit's own rounds;
//   duo  (sg_warp_ag_rows_banded_duo): unit (row i, segment j) at step i + j, two units per step, the longer of their loops.
// Built and driven by tools/narrow_band_counts.py.
#include <stdint.h>
#include <string.h>
#include <vector>

static void nb_call(bool banded, int numVec, int w, int patternLen, int textLen);
static void nb_unit(int row, int seg, int nVecHere, int rounds);
#define SG_AG_CALL_HOOK(banded, numVec, w, patternLen, textLen) nb_call(banded, numVec, w, patternLen, textLen)
#define SG_AG_UNIT_HOOK(row, seg, nVecHere, rounds) nb_unit(row, seg, nVecHere, rounds)
#include "../tests/hostsim/hostsim.cpp"

enum {
    NB_CALLS, NB_UNITS, NB_ROWS, NB_ROUNDS_ROWS, NB_STEPS_DUO, NB_ROUNDS_DUO, NB_STEPS_ONE_UNIT,
    NB_CALLS_NUMVEC = 8,                 // [numVec 1..4] at 8 + numVec - 1
    NB_UNITS_NUMVEC = 12,
    NB_CALLS_W = 16,                     // [w 0..15]
    NB_UNITS_NVECHERE = 32,              // [nVecHere 0..4]
    NB_ROUNDS_HIST = 40,                 // [rounds 1..7] of the units
    NB_N = 48
};
static int64_t g_nb[NB_N];
static bool g_narrow = false;
static std::vector<int> g_stepRounds, g_stepUnits;      // per duo step of the current call: longest loop, units
static int g_lastRow = -1, g_numVec = 0;

static void nb_flush()
{
    if (!g_narrow) return;
    for (size_t t = 0; t < g_stepRounds.size(); t++) {
        g_nb[NB_STEPS_DUO]++;
        g_nb[NB_ROUNDS_DUO] += g_stepRounds[t];
        if (g_stepUnits[t] == 1) g_nb[NB_STEPS_ONE_UNIT]++;
    }
    g_stepRounds.clear(); g_stepUnits.clear();
    g_narrow = false;
}

static void nb_call(bool banded, int numVec, int w, int patternLen, int textLen)
{
    (void)patternLen; (void)textLen;
    nb_flush();
    g_narrow = banded && numVec <= 4;
    g_lastRow = -1; g_numVec = numVec;
    if (!g_narrow) return;
    g_nb[NB_CALLS]++;
    g_nb[NB_CALLS_NUMVEC + numVec - 1]++;
    if (w >= 0 && w < 16) g_nb[NB_CALLS_W + w]++;
}

static void nb_unit(int row, int seg, int nVecHere, int rounds)
{
    if (!g_narrow) return;
    g_nb[NB_UNITS]++;
    g_nb[NB_UNITS_NUMVEC + g_numVec - 1]++;
    if (row != g_lastRow) { g_nb[NB_ROWS]++; g_lastRow = row; }
    g_nb[NB_ROUNDS_ROWS] += rounds;
    if (nVecHere >= 0 && nVecHere <= 4) g_nb[NB_UNITS_NVECHERE + nVecHere]++;
    if (rounds >= 1 && rounds <= 7) g_nb[NB_ROUNDS_HIST + rounds - 1]++;
    const size_t t = (size_t)(row + seg);
    if (g_stepRounds.size() <= t) { g_stepRounds.resize(t + 1, 0); g_stepUnits.resize(t + 1, 0); }
    if (rounds > g_stepRounds[t]) g_stepRounds[t] = rounds;
    g_stepUnits[t]++;
}

extern "C" {
void nb_reset(void) { nb_flush(); memset(g_nb, 0, sizeof(g_nb)); }
void nb_counts(int64_t *out) { nb_flush(); memcpy(out, g_nb, sizeof(g_nb)); }
int nb_size(void) { return NB_N; }
}
