// warpsim.cpp -- TEST-ONLY: the warp-cooperative affine-gap forms (snap_b200/csrc/sg_warp_ag*.cuh), compiled for the host on the
// 32-lane SIMT emulator of warpsim.h.  Built into tests/_build/libwarpsim.so by tests/warpsim_lib.py; never loaded by the product.
#include <string>
#include <math.h>
#include <limits.h>
#include <stddef.h>
#include "warpsim.h"
#include "../../snap_b200/csrc/sg_ag.h"
#include "../../snap_b200/csrc/sg_host.h"
#include "../../snap_b200/csrc/sg_warp_ag.cuh"

namespace ws {

thread_local Warp *g_warp = nullptr;

#if defined(__x86_64__)
// void ws_switch(void **saveSp, void *newSp): park the caller (callee-saved registers on its own stack), continue on newSp
asm(R"(
.text
.globl ws_switch
.type ws_switch,@function
ws_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size ws_switch,.-ws_switch
)");
#else
#error "warpsim: only x86-64 has a context switch here"
#endif

static void lane_entry()
{
    Warp *w = g_warp;
    const int lane = w->current;
    w->body(lane);
    w->lanes[lane].done = true;
    w->lanes[lane].op = OP_DONE;
    void *dummy;
    ws_switch(&dummy, w->mainSp);
    abort();
}

uint64_t park(int op, unsigned mask, uint64_t val, int arg)
{
    Warp *w = g_warp;
    Lane &L = w->lanes[w->current];
    L.op = op; L.mask = mask; L.val = val; L.arg = arg;
    ws_switch(&L.sp, w->mainSp);
    return L.result;
}

static void resolve(Warp *w)
{
    int op = OP_NONE;
    unsigned alive = 0;
    for (int l = 0; l < 32; l++) {
        if (w->lanes[l].done) continue;
        alive |= 1u << l;
        if (op == OP_NONE) op = w->lanes[l].op;
        else if (op != w->lanes[l].op) { fprintf(stderr, "warpsim: lanes parked at different primitives (%d vs %d at lane %d): divergent code around a warp-synchronous call\n", op, w->lanes[l].op, l); abort(); }
    }
    for (int l = 0; l < 32; l++) {
        if (!(alive >> l & 1)) continue;
        Lane &L = w->lanes[l];
        if (!(L.mask >> l & 1)) { fprintf(stderr, "warpsim: lane %d not in its own mask %08x\n", l, L.mask); abort(); }
        if (L.mask & ~alive) { fprintf(stderr, "warpsim: mask %08x names exited lanes (alive %08x)\n", L.mask, alive); abort(); }
        const unsigned m = L.mask;
        switch (op) {
        case OP_SHFL: { const int s = L.arg & 31; L.result = (m >> s & 1) ? w->lanes[s].val : L.val; break; }       // (reading a lane outside the mask is undefined on the device)
        case OP_SHFL_UP: { const int s = l - L.arg; L.result = (s >= 0) ? w->lanes[s].val : L.val; break; }
        case OP_SHFL_DOWN: { const int s = l + L.arg; L.result = (s < 32) ? w->lanes[s].val : L.val; break; }
        case OP_SHFL_XOR: { const int s = (l ^ L.arg) & 31; L.result = w->lanes[s].val; break; }
        case OP_BALLOT: { unsigned r = 0; for (int k = 0; k < 32; k++) if ((m >> k & 1) && w->lanes[k].val) r |= 1u << k; L.result = r; break; }
        case OP_REDUCE_MAX_S: { int r = INT_MIN; for (int k = 0; k < 32; k++) if (m >> k & 1) { int v = (int)(uint32_t)w->lanes[k].val; if (v > r) r = v; } L.result = (uint32_t)r; break; }
        case OP_REDUCE_MIN_S: { int r = INT_MAX; for (int k = 0; k < 32; k++) if (m >> k & 1) { int v = (int)(uint32_t)w->lanes[k].val; if (v < r) r = v; } L.result = (uint32_t)r; break; }
        case OP_REDUCE_MAX_U: { unsigned r = 0; for (int k = 0; k < 32; k++) if (m >> k & 1) { unsigned v = (unsigned)w->lanes[k].val; if (v > r) r = v; } L.result = r; break; }
        case OP_REDUCE_ADD: { unsigned r = 0; for (int k = 0; k < 32; k++) if (m >> k & 1) r += (unsigned)w->lanes[k].val; L.result = r; break; }
        case OP_REDUCE_OR: { unsigned r = 0; for (int k = 0; k < 32; k++) if (m >> k & 1) r |= (unsigned)w->lanes[k].val; L.result = r; break; }
        case OP_REDUCE_AND: { unsigned r = ~0u; for (int k = 0; k < 32; k++) if (m >> k & 1) r &= (unsigned)w->lanes[k].val; L.result = r; break; }
        case OP_SYNC: L.result = 0; break;
        default: fprintf(stderr, "warpsim: bad op %d\n", op); abort();
        }
    }
    w->syncOps++;
}

void run_warp(const std::function<void(int)> &body, size_t stackBytes)
{
    Warp w;
    memset(w.lanes, 0, sizeof(w.lanes));
    w.body = body; w.syncOps = 0;
    Warp *outer = g_warp;
    g_warp = &w;
    for (int l = 0; l < 32; l++) {
        Lane &L = w.lanes[l];
        L.stack = (uint8_t *)malloc(stackBytes);
        uintptr_t top = ((uintptr_t)L.stack + stackBytes) & ~(uintptr_t)15;
        void **sp = (void **)top;
        *--sp = nullptr;                       // fake return address of lane_entry: keeps rsp = 8 mod 16 at its entry
        *--sp = (void *)&lane_entry;
        for (int r = 0; r < 6; r++) *--sp = nullptr;
        L.sp = sp;
    }
    for (;;) {
        int live = 0;
        for (int l = 0; l < 32; l++) {
            if (w.lanes[l].done) continue;
            w.current = l;
            ws_switch(&w.mainSp, w.lanes[l].sp);
            if (!w.lanes[l].done) live++;
        }
        if (!live) break;
        resolve(&w);
    }
    for (int l = 0; l < 32; l++) free(w.lanes[l].stack);
    g_warp = outer;
}

} // namespace ws

static void make_scratch(const SgParams &p, std::vector<uint8_t> &mem, SgScratch *s)
{
    mem.assign(sg_scratch_bytes(p) + 256, 0);
    uint8_t *base = (uint8_t *)(((uintptr_t)mem.data() + 255) & ~(uintptr_t)255);
    sg_scratch_carve(p, base, s);
}

static const uint32_t WS_MAX_READ_LEN = 1000;         // the scratch of the emulated warp, like the device leaf tests' (leaf_scratch)

extern "C" {

// sg_ag_small_scores for a scoring scheme (the reference's order: match, sub, open, extend, 5', 3'), at the emulated warp's maxReadLen:
// whether the alignment kernels would take the specialised forms (packed rows, narrow-band rows) under it.
int ws_ag_small_scores(const snapgpu_ag_params *ap)
{
    SgAgParams P = sg_ag_params(ap->matchReward, ap->subPenalty, ap->gapOpenPenalty, ap->gapExtendPenalty, ap->fivePrimeEndBonus, ap->threePrimeEndBonus);
    return sg_ag_small_scores(P, WS_MAX_READ_LEN) ? 1 : 0;
}

// Same contract as hostsim's hs_ag_batch / the ABI's snapgpu_test_ag_warp: one emulated warp runs the jobs in order (so the
// traceback array carries over from job to job like the reference's).  usePacked: SgAgParams.usePacked (0 int forms, 1 packed, 2 unrolled packed;
// + 4: the experimental narrow-band form of sg_warp_ag_duo.cuh, + 8: with its per-round H in the arena instead of the shared-memory block).
long long ws_ag_batch(const snapgpu_ag_params *ap, const char *textBuf, const char *patBuf, const char *qualBuf, const snapgpu_ag_job *jobs,
                      int64_t nJobs, snapgpu_ag_out *out, int usePacked)
{
    static SgTables T; static bool init = false;
    if (!init) { sg_init_tables(T, 20); init = true; }
    SgParams p; memset(&p, 0, sizeof(p));
    p.poolSize = 1; p.tableSlots = 2; p.numWeightLists = 2; p.maxReadLen = WS_MAX_READ_LEN;
    std::vector<uint8_t> mem; SgScratch s; make_scratch(p, mem, &s);
    static SgWarpSmall small;                    // the per-warp shared-memory block of the alignment kernels
    if (usePacked & 8) { usePacked &= ~8; }      // 8: without it (the arena copies are used, as in the leaf test kernel)
    else { s.lvLs = small.lvL; s.lvAs = small.lvA; s.lvSmallCells = SG_SMALL_LV_CELLS; s.agSnap = (uint32_t *)small.lvL; }
    SgAgParams P = sg_ag_params(ap->matchReward, ap->subPenalty, ap->gapOpenPenalty, ap->gapExtendPenalty, ap->fivePrimeEndBonus, ap->threePrimeEndBonus);
    P.usePacked = usePacked;
    long long ops = 0;
    for (int64_t j = 0; j < nJobs; j++) {
        SgAgResult res[32];
        ws::Warp *before = ws::g_warp; (void)before;
        ws::run_warp([&](int lane) {
            SgAgResult &r = res[lane];
            r.agScore = -1; r.textOffset = 0; r.patternOffset = 0; r.nEdits = 0; r.matchProbability = 0.0;
            sg_warp_ag_compute<3>(T, s, P, jobs[j].dir, jobs[j].banded != 0, (const uint8_t *)textBuf + jobs[j].textOff, jobs[j].textLen,
                                  (const uint8_t *)patBuf + jobs[j].patOff, (const uint8_t *)qualBuf + jobs[j].patOff, jobs[j].patternLen, jobs[j].w,
                                  jobs[j].scoreInit, jobs[j].isRC != 0, jobs[j].useClippingOptimizations != 0, &r, lane);
            __syncwarp();
        });
        for (int l = 1; l < 32; l++) {
            if (memcmp(&res[l], &res[0], sizeof(SgAgResult)) != 0 && !(res[l].agScore == res[0].agScore && res[l].textOffset == res[0].textOffset &&
                res[l].patternOffset == res[0].patternOffset && res[l].nEdits == res[0].nEdits && res[l].matchProbability == res[0].matchProbability)) {
                fprintf(stderr, "warpsim: job %lld: lane %d disagrees with lane 0\n", (long long)j, l); abort();
            }
        }
        out[j].agScore = res[0].agScore; out[j].textOffset = res[0].textOffset; out[j].patternOffset = res[0].patternOffset; out[j].nEdits = res[0].nEdits;
        out[j].matchProbability = res[0].matchProbability;
    }
    return ops;
}

} // extern "C"
