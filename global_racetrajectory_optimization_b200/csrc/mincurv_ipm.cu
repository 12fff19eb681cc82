// K2b -- box-constrained QP solve  min 1/2 a^T H a + f^T a,  lb <= a <= ub  by a Mehrotra predictor-corrector
// primal-dual interior-point method (replaces quadprog.solve_qp inside tph.opt_min_curv, call site
// main_globaltraj.py:264-271; SURVEY.md A.3), and K2b' -- the same iteration with tph's curvature rows.
//
// One CTA of two warps per QP instance, eight CTAs per SM.  H is the cyclic band (half-bandwidth 32) assembled by K2a.
// Every interior-point iteration factorises M = H + D (D diagonal, from the barrier) as a bordered LDL^T:
//   chain nodes 0..NA-1 (NA = n - 32):  A = M[chain, chain] = L D L^T   (banded, L unit lower, 32 sub-diagonals)
//   separator = the last 32 nodes (they close the cycle):  G = Y L^-T,  Y = M[sep, chain]  (the fill row of the separator)
//                                                          S = M[sep, sep] - G D^-1 G^T = L_S D_S L_S^T
// column by column, right-looking, with the whole active window in REGISTERS:
//   warp 0 (chain): lane = row (rows k+1..k+32 of the window, circular), 32 accumulators per lane = the updates of
//           the row's 32 window columns.  Step k: v = A[row][k] - acc[0]; the column is broadcast through shared memory;
//           w = 1/d_k; l = v w; acc[c] <- acc[c+1] + l v_c (32 independent DFMAs: the register file is the sliding window,
//           the slide is the operand index, no moves).  The forward substitution of the predictor's right-hand side rides
//           along (one more accumulator).  The pivot chain per column is DADD -> STS/LDS -> rcp -> DMUL -> DFMA.
//   warp 1 (fill):  lane = separator row, 32 accumulators = the updates of G[row][k+1..k+32]; consumes warp 0's columns
//           from a shared-memory ring eight columns behind, and accumulates S -= (G w) G^T on the FP64 tensor cores
//           (mma.sync.m8n8k4.f64, SASS DMMA) once per eight columns.
// The first version of this kernel ran a 32x32-block Cholesky on DMMA with explicit block inverses: a small share of the
// fp64 pipe, latency-bound on the in-block pivot chains and on the hand-offs between three warp roles.  Here every step offers 64 independent DFMAs per instance and eight
// instances share an SM, so the fp64 pipe and the issue slots are what is busy.
//
// The factor (per column: the 32 band entries of L + w, the 32 entries of G + w) goes to the instance's HBM slab and
// is streamed back by the triangular sweeps through a shared-memory ring of 8-column units filled by cp.async.bulk
// (TMA, 1-D) on mbarriers -- the band rows of H reach warp 0 the same way.  Per iteration: factor written once, read
// three times (the predictor's forward sweep is fused into the factorisation).
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include "capi.cuh"
#include "mincurv_ops.cuh"

namespace mc {

constexpr unsigned FULL = 0xffffffffu;
constexpr int IP_THREADS = 64;
constexpr int SUB = 8;                 // columns per hand-off / streaming unit
constexpr int VBP = 12;                // pitch of the row-major panel buffers (conflict-free DMMA fragment loads, 16-byte rows)
constexpr int FROW = 33;               // pitch of a fill row: [g (32), w]
constexpr int HB_SLOTS = 2;            // band-row units of warp 0 (the next panel's is in flight)
constexpr int HO_SLOTS = 2;            // panels between warp 0 and warp 1
constexpr int LROW = 33;               // pitch of a chain-factor column: its 32 band entries of [Q - I; L21], w (see lt_slot)
#ifndef MC_LT_SLOTS
#define MC_LT_SLOTS 3
#endif
constexpr int LT_SLOTS = MC_LT_SLOTS;  // sweep rings: warp 0 streams the chain rows (LT), warp 1 the fill rows (GT), concurrently
constexpr int GT_SLOTS = 6 - LT_SLOTS;
constexpr int RING_UNITS = LT_SLOTS + GT_SLOTS;       // mbarriers: [0, LT_SLOTS) warp 0, [LT_SLOTS, RING_UNITS) warp 1
constexpr int QDEPTH = 16;             // units of z (forward) / t (backward) in flight between the two warps
constexpr int LT_UNIT_DOUBLES = SUB * LROW;           // 264 (2112 bytes: one bulk copy, 16-byte multiple)
constexpr int GT_UNIT_DOUBLES = SUB * FROW;           // 264 (2112 bytes, like a chain unit)
constexpr unsigned HB_UNIT_BYTES = SUB * HB_PITCH * sizeof(double);   // 2176

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}

// ---- TMA (bulk async copy) + mbarrier helpers ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
#ifndef MC_WAIT_MODE
#define MC_WAIT_MODE 1
#endif
#ifndef MC_RELAXED_BACKOFF_NS
#define MC_RELAXED_BACKOFF_NS 250
#endif

// MC_WAIT_MODE 0: try_wait with a long suspend hint (the thread is parked until the phase completes);
//              1: test_wait spin (non-blocking probe): the waiter resumes within a few cycles of the arrival.
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
#if MC_WAIT_MODE == 0
    asm volatile("{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, 0x989680;\n"
                 " @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
#else
    asm volatile("{\n .reg .pred p;\n WAIT_%=:\n mbarrier.test_wait.parity.shared::cta.b64 p, [%0], %1;\n"
                 " @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
#endif
}
// same, for the warp that is normally AHEAD of its producer (the fill warp, ~20 % of its time): parked by the hardware
// (try_wait with a suspend hint) instead of probing -- the probes of the spin version were 16 % of all executed instructions
// and took issue slots from the chain warps of the same scheduler; runs with them fell into a slow mode now and then.
// -DMC_RELAXED_SPIN_NS=<ns> restores the probing loop with that back-off, for experiments.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t *bar, unsigned parity) {
#ifndef MC_RELAXED_SPIN_NS
    // (one try_wait parks the warp for well under a microsecond before it reports "not yet": the back-off between two
    //  of them keeps the probes of a ~1400-cycle wait at a handful instead of ~200)
    unsigned ok = 0;
    for (;;) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, 0x989680;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (ok) break;
        __nanosleep(MC_RELAXED_BACKOFF_NS);
    }
#else
    unsigned ok = 0;
    for (;;) {
        asm volatile("{\n .reg .pred p;\n mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (ok) break;
        __nanosleep(MC_RELAXED_SPIN_NS);
    }
#endif
}
// The factor is a stream (written once, read three times per iteration, 0.5 MB per instance, far beyond what L2 can
// keep for the 1056 resident instances of an H100): its bulk stores and loads carry an evict-first L2 policy so that they
// do not push the O(N) iterate vectors of the interior-point loop out of L2.
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// The band rows of H are read, not streamed: with shared centre lines every instance of a centre line reads the owner's
// band (32 bands, 8.7 MB, for the 2112 instances of the headline batch), so they keep the normal policy and stay in L2.
__device__ __forceinline__ uint64_t l2_evict_normal_policy() {
    uint64_t pol;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ void tma_load_1d(void *dst, const void *src, unsigned bytes, uint64_t *bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
// A factor unit is written into a shared-memory staging buffer and leaves it as one bulk store (bulk-group completion):
// every sector of the unit reaches L2 whole and at once, instead of two or three partial writes per sector from
// per-lane stores at different moments.  The writing lanes run fence_proxy_async_smem() and the warp __syncwarp() before
// one lane issues the store; that lane runs bulk_wait_read() (then the warp __syncwarp()) before the buffer is written
// again, and bulk_wait() before the units are read back.
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_store_1d(void *dst, const void *src, unsigned bytes, uint64_t policy) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;\n"
                 "cp.async.bulk.commit_group;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes), "l"(policy) : "memory");
}
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// cycle counters of the instrumented build (-DMC_PROFILE), accumulated by CTA 0 and read by mc_debug_read_profile; slots
// 3, 4 and 16 are not written.  tools/prof_run.py names the slots in this order.
enum ProfSlot {
    PROF_UPDATE = 0,                                     // update pass: step, residuals, next barrier diagonal and rhs
    PROF_CHAIN = 1,                                      // factor_chain (warp 0)
    PROF_FWD_SWEEPS = 2,                                 // sweep_forward + sweep_sep_rhs (corrector; the predictor's is fused)
    PROF_SEP_LDLT = 5,                                   // separator block and its LDL^T
    PROF_SOLVE_PRED = 6, PROF_SOLVE_CORR = 7,            // solve: predictor, corrector
    PROF_BWD_SWEEPS = 8,                                 // sweep_sep_solve + sweep_backward
    PROF_TOTAL = 9, PROF_FACTOR = 10,                    // whole instance; factor
    PROF_NQP = 11, PROF_ITERS = 12,                      // counts: instances, interior-point iterations
    PROF_FILL = 13,                                      // factor_fill (warp 1)
    PROF_W0_WAIT_HB = 14,                                // warp 0 waiting for the band rows of H
    PROF_STEPLEN = 15,                                   // corrector step lengths
    PROF_AFFINE = 17, PROF_CORR_RHS = 18,                // affine step lengths and centring; corrector right-hand side
    PROF_W0_WAIT_HO_EMPTY = 19, PROF_W1_WAIT_HO_FULL = 20,   // hand-off waits: warp 0 for a free slot, warp 1 for a panel
    PROF_W1_UPDATE = 21,                                 // warp 1: trailing update of G and S
    PROF_RING_WAIT_W0 = 22, PROF_RING_WAIT_W1 = 23,      // sweep ring waits: warp 0 (chain units), warp 1 (fill units)
    PROF_SLOTS = 24
};
#ifdef MC_PROFILE
__device__ unsigned long long g_prof[PROF_SLOTS];
#define PROF_T0(name) const long long name = clock64()
#define PROF_ADD(slot, t0) do { if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&g_prof[slot], (unsigned long long)(clock64() - (t0))); } while (0)
#define PROF_ADD1(slot, t0) do { if (blockIdx.x == 0 && threadIdx.x == 32) atomicAdd(&g_prof[slot], (unsigned long long)(clock64() - (t0))); } while (0)
__device__ unsigned long long g_seg[32];
#ifdef MC_PROFILE_SEG      // per-panel sub-phase marks: ~200 cycles each, only for attributing time inside one panel
#define SEG_BEGIN() long long _seg_t = clock64()
#define SEG(slot) do { if (blockIdx.x == 0 && (threadIdx.x & 31) == 0) { const long long _n = clock64(); atomicAdd(&g_seg[slot], (unsigned long long)(_n - _seg_t)); _seg_t = _n; } } while (0)
#else
#define SEG_BEGIN() do { } while (0)
#define SEG(slot) do { } while (0)
#endif
#else
#define SEG_BEGIN() do { } while (0)
#define SEG(slot) do { } while (0)
#define PROF_T0(name) do { } while (0)
#define PROF_ADD(slot, t0) do { } while (0)
#define PROF_ADD1(slot, t0) do { } while (0)
#endif

// 1/d for a positive, normal d: hardware seed (rcp.approx.f64, ~20 bits) + two Newton steps (relative error ~1e-16).
// Four dependent DFMAs instead of the IEEE division routine with its special-case path: the pivot chain of the
// factorisation is latency bound on exactly this.
__device__ __forceinline__ double fast_rcp(double d) {
    double x;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(x) : "d"(d));
    double e = fma(-d, x, 1.0);
    x = fma(x, e, x);
    e = fma(-d, x, 1.0);
    return fma(x, e, x);
}

// one panel (eight columns) handed from warp 0 to warp 1
struct Handoff {
    double vb[32 * VBP];       // L of the window rows k0+8 .. k0+39 x the panel's 8 columns, row-major (DMMA fragments)
    double l11[64];            // the panel's unit-lower diagonal block, row-major [m][j] (m > j used)
    double w[8], y[8];         // 1/d and the forward-substituted right-hand side of the panel's columns
};

struct IpShared {
    union {
        struct {
            double hb[HB_SLOTS][SUB * HB_PITCH];      // band rows of H staged for warp 0 (TMA)
            Handoff ho[HO_SLOTS];                     // warp 0 -> warp 1
            double gb[32 * VBP];                      // warp 1: the panel of the fill rows, row-major (DMMA fragments)
            double gt[GT_UNIT_DOUBLES];               // warp 1: the panel's fill unit, staged for its bulk store
        } f;
        struct {
            double lt[LT_SLOTS][LT_UNIT_DOUBLES];     // sweeps: streamed chain units (warp 0)
            double gt[GT_SLOTS][GT_UNIT_DOUBLES];     //         streamed fill units (warp 1)
            double q[QDEPTH * SUB];                   //         z (forward) / t (backward) handed between the warps
        } sw;
        double win[hband_win_doubles(IP_THREADS)];    // K2b': scratch of the weighted band assembly
    } u;
    union {
        double Ss[32 * 33];                           // separator block -> its L_S (strictly lower, in place)
        struct {
            double sfrag[20 * 32];                    // during the chain: S accumulators (DMMA C fragments, [block][lane][2])
            double lt[LT_UNIT_DOUBLES];               // during the chain: warp 0's chain unit of the panel, staged for its bulk store
        } c;
    } s;
    double wS[32], gs[32], part[2][32];
    double red[32];
    uint64_t hb_full[HB_SLOTS], ho_full[HO_SLOTS], ho_empty[HO_SLOTS], ring_full[RING_UNITS];
    unsigned ring_phase[2];                           // parity bit per ring slot, one word per warp
    int prog[4];                                      // sweep progress (units done): forward w0, w1; backward w0, w1
    int flag;
    int next;                                         // next instance index (dynamic work distribution)
    int resumed;                                      // ... a parked one (sliced schedule of mincurv_pdip_kernel)
};
static_assert(offsetof(IpShared, s.c.lt) % 16 == 0 && offsetof(IpShared, u.f.gt) % 16 == 0,
              "the sources of the factor's bulk stores must be 16-byte aligned");
static_assert(sizeof(IpShared::s) == 32 * 33 * sizeof(double), "the chain unit's staging must fit beside the S accumulators");

// pointers into the instance slab that the factorisation and the sweeps use.  Factor rows in HBM, one bulk copy per unit
// of eight rows (every unit 16-byte aligned):
//   LT[k0+j] = [ 32 band entries of column j of [Q - I; L21], w_k ]   (pitch 33) the chain factor, one panel of columns
//              k0 .. k0+7 at a time: L21 = the 32 rows of L below the panel, Q = L11^-1 the inverse of the panel's
//              unit-lower block, so that the panel's triangular solve in the sweeps is a mat-vec too (forward: y1 = Q a1,
//              a2 -= L21 y1; backward: u = t1 - L21^T x2, x1 = Q^T u).  w = 1/d_k.  With the rows m = 0..39 of
//              [Q - I; L21] counted from k0, column j is nonzero for j < m <= j + 32 only (Q - I strictly lower, L with 32
//              sub-diagonals): exactly 32 entries, kept at lt_slot(j, m).  The sweeps set the other entries to zero by predicate
//   GT[k]    = [ G[0 .. 31][k],  w_k ]                        (pitch 33)
// so warp 0's sweeps read nothing but the streamed units (no per-column global loads on the serial chains).  z = w y, what
// the separator's part of the backward half needs, is a vector of its own behind GT: the forward half of every solve
// writes it, eight adjacent columns per store (full sectors); inside the fill rows it was an 8-byte store into each
// 264-byte row long after the row had been written.  Columns NA .. 8 ceil(NA / 8) - 1 are padding (pivot 1, nothing
// else): every unit is a full panel.
struct Factor {
    const double *HB;      // band of H, row i: H[i][i .. i+32] (read only: possibly another instance's, shared centre lines)
    const double *DD;      // barrier diagonal
    double *LT, *GT, *Z;
    int NA;
};

__device__ __forceinline__ Factor make_factor(double *slab, const Layout &L, int n, const double *HB) {
    double *LT = slab + L.o_tiles, *GT = LT + (size_t)L.np * LROW;
    return {HB, vec(slab, L, V_DD), LT, GT, GT + (size_t)L.np * FROW, n - 32};
}

// slot of entry (c, m), c < m <= c + 32, in a chain unit: the packed order m - c - 1 rotated by 4 c, so that the sweeps'
// DMMA fragment loads (a column quartet x eight rows, or eight columns x a row quartet) fall on distinct shared-memory banks
__device__ __forceinline__ int lt_slot(int c, int m) { return LROW * c + ((m + 3 * c - 1) & 31); }
__device__ __forceinline__ double lt_entry(const double *unit, int c, int m) {
    return (c < m && m <= c + 32) ? unit[lt_slot(c, m)] : 0.0;
}

__device__ __forceinline__ int blk(int I, int J) { return (I * (I + 1)) / 2 + J; }      // lower 8x8 block (I >= J) of a 4x4 block grid

// ---- warp 0: LDL^T of the chain, one panel of eight columns at a time, with the forward substitution of g fused in.
//      The 32x32 window of accumulated updates (rows/columns k0 .. k0+31, lower blocks) lives in DMMA C fragments.
//      Panel step: (1) block column 0 -> row layout (lane l = row k0 + l; lanes 0..7 also carry the entering row
//      k0 + 32 + l); (2) eight pivots: d_j by shuffle from lane j, w = 1/d, l = v w, v_{j',j} by shuffle from lane j'
//      for the in-panel updates; (3) trailing update W'[I][J] = W[I+1][J+1] + (L d)(L)^T on the tensor cores, which also
//      slides the window by one block (the block row of the eight entering rows starts from zero). ----
__device__ __noinline__ bool factor_chain(IpShared &sh, const double *__restrict__ HBp, const double *__restrict__ DD, double *__restrict__ LTp, const int NA, const double *__restrict__ g, unsigned tick) {
    const int lane = threadIdx.x & 31;
    const int gq = lane >> 2, q = lane & 3;
    const int nunits = (NA + SUB - 1) / SUB;
    const uint64_t pol = l2_evict_normal_policy();
    double *lst = sh.s.c.lt;                           // the panel's unit, at its offsets in LT
    double W[10][2];
#pragma unroll
    for (int b = 0; b < 10; ++b) { W[b][0] = 0.0; W[b][1] = 0.0; }
    // right-hand side: gv = g - (L y so far) of row k0 + lane; the entering rows take their g from a block of 32 loaded a
    // block ahead (a load issued inside the panel step would be waited for right away: the scoreboard is per warp).
    // The barrier diagonal of the panel's own rows comes the same way: ddcur = D of the current block of 32 rows.
    double gv = (lane < NA) ? g[lane] : 0.0;
    double gcur = (32 + lane < NA) ? g[32 + lane] : 0.0;
    double gnext = (64 + lane < NA) ? g[64 + lane] : 0.0;
    double ddcur = (lane < NA) ? DD[lane] : 0.0;
    double ddnext = (32 + lane < NA) ? DD[32 + lane] : 0.0;
    bool ok = true;
    if (lane == 0) {
        mbar_expect_tx(&sh.hb_full[tick % HB_SLOTS], HB_UNIT_BYTES);
        tma_load_1d(sh.u.f.hb[tick % HB_SLOTS], HBp, HB_UNIT_BYTES, &sh.hb_full[tick % HB_SLOTS], pol);
    }
    SEG_BEGIN();
    for (int t = 0; t < nunits; ++t) {
        const unsigned ht = tick + t, hs = ht % HB_SLOTS, ls = ht % HO_SLOTS;
        const int k0 = t * SUB;
        SEG(8);
        if (t > 0 && (t & 3) == 0) {                  // a new block of 32 rows enters over the next four panels
            gcur = gnext;
            ddcur = ddnext;
            const int idx = k0 + 64 + lane, idd = k0 + 32 + lane;
            gnext = (idx < NA) ? g[idx] : 0.0;
            ddnext = (idd < NA) ? DD[idd] : 0.0;
        }
        if (lane == 0 && t + 1 < nunits) {            // band rows of the next panel (slot of panel t-1: all lanes are past it)
            const unsigned h2 = (ht + 1) % HB_SLOTS;
            mbar_expect_tx(&sh.hb_full[h2], HB_UNIT_BYTES);
            tma_load_1d(sh.u.f.hb[h2], HBp + (size_t)(t + 1) * SUB * HB_PITCH, HB_UNIT_BYTES, &sh.hb_full[h2], pol);
        }
        PROF_T0(tw1);
        if (ht >= (unsigned)HO_SLOTS) mbar_wait(&sh.ho_empty[ls], ((ht / HO_SLOTS) - 1u) & 1u);
        PROF_ADD(PROF_W0_WAIT_HO_EMPTY, tw1);
        Handoff &ho = sh.u.f.ho[ls];
        SEG(9);
        // ---- (1) block column 0 of the window -> row layout, through the (still free) fragment area of the hand-off slot
#pragma unroll
        for (int I = 0; I < 4; ++I)
            *reinterpret_cast<double2 *>(&ho.vb[(8 * I + gq) * VBP + 2 * q]) = make_double2(W[blk(I, 0)][0], W[blk(I, 0)][1]);
        __syncwarp();
        double p[8], p2[8];
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            const double2 uu = *reinterpret_cast<const double2 *>(&ho.vb[lane * VBP + j]);
            p[j] = uu.x; p[j + 1] = uu.y;
        }
        const double ddl = __shfl_sync(FULL, ddcur, ((t & 3) << 3) + (lane & 7));     // lanes 0..7: D of row k0 + lane
        PROF_T0(tw0);
        mbar_wait(&sh.hb_full[hs], (ht / HB_SLOTS) & 1u);
        PROF_ADD(PROF_W0_WAIT_HB, tw0);
        const double *hbg = sh.u.f.hb[hs];
        const bool row_ok = (k0 + lane < NA), row2_ok = (lane < 8) && (k0 + 32 + lane < NA);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int d = lane - j;                    // row k0 + lane, column k0 + j: band entry H[k0+j][d]; d = 0: the pivot (with D)
            const bool col_ok = (k0 + j < NA);
            double a1 = 0.0;
            if (d >= 0 && row_ok && col_ok) {
                a1 = hbg[j * HB_PITCH + d];
                if (d == 0) a1 += ddl;
            }
            if (d == 0 && !col_ok) a1 = 1.0;           // padding column: unit pivot
            p[j] = (d >= 0) ? a1 - p[j] : 0.0;
            const int d2 = 32 + lane - j;              // entering row k0 + 32 + lane: nonzero for j >= lane only, no updates yet
            p2[j] = (row2_ok && col_ok && d2 <= 32) ? hbg[j * HB_PITCH + d2] : 0.0;
        }
        double gv2 = __shfl_sync(FULL, gcur, ((t & 3) << 3) + (lane & 7));
        if (lane >= 8) gv2 = 0.0;
        if (lane == 0) bulk_wait_read();               // the previous panel's unit has left the staging buffer
        __syncwarp();                                  // every lane has read its row of block column 0: the slot can take L now
        SEG(10);
        // ---- (2) the panel ----
        double dsave = 1.0, wsave = 1.0, ysave = 0.0;
        const int wr = (lane >= 8) ? lane - 8 : 24 + lane;      // window row (after the slide) of the row this lane hands over
        // the eight slots lt_slot(j, 8 + wr) of this lane's L21 entries, recomputed in every panel: hoisted out of the loop
        // they took eight registers and made the loop spill
        int wrs;
        asm volatile("mov.b32 %0, %1;" : "=r"(wrs) : "r"(wr));
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const double dj = __shfl_sync(FULL, p[j], j);
            const double yj = __shfl_sync(FULL, gv, j);
            if (!(dj > 0.0)) ok = false;
            const double w = fast_rcp(dj);
            const double lt = p[j] * w, lt2 = p2[j] * w;           // (lanes <= j: lt is not an entry of L; lanes > j: lt2 = 0)
            ho.vb[wr * VBP + j] = (lane >= 8) ? lt : lt2;
            if (lane >= 8 || lane <= j) lst[lt_slot(j, 8 + wrs)] = (lane >= 8) ? lt : lt2;      // L21: the band of the 32 rows below the panel
            if (lane < 8 && lane > j) ho.l11[lane * 8 + j] = lt;
            if (lane == j) { dsave = dj; wsave = w; ysave = yj; }
            gv = fma(-lt, yj, gv);                                 // (lanes <= j: gv is dead)
            gv2 = fma(-lt2, yj, gv2);
#pragma unroll
            for (int jj = j + 1; jj < 8; ++jj) {
                const double vj = __shfl_sync(FULL, p[j], jj);     // v of row k0 + jj in column j (unscaled)
                p[jj] = fma(-lt, vj, p[jj]);
                p2[jj] = fma(-lt2, vj, p2[jj]);
            }
        }
        SEG(11);
        if (lane < 8) {
            ho.w[lane] = wsave;
            ho.y[lane] = ysave;
        }
        __syncwarp();
        // ---- (2b) Q = L11^-1 (the panel's unit-lower block): with it the panel's triangular solves in the sweeps are mat-vecs.
        //      column j of the unit: the strictly lower part of Q's column j, L21's (stored above), w ----
        {
            const int jq = lane & 7;
            double q8[8];
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                double sacc = (m == jq) ? 1.0 : 0.0;
#pragma unroll
                for (int i = 0; i < m; ++i) sacc = fma(-ho.l11[m * 8 + i], q8[i], sacc);
                q8[m] = sacc;
            }
            if (lane < 8) {
                double *ltq = lst + 36 * lane - 1;     // + m = lt_slot(lane, m) for the rows m < 8 of Q (no wrap)
#pragma unroll
                for (int m = 1; m < 8; ++m)
                    if (m > lane) ltq[m] = q8[m];
                lst[lane * LROW + 32] = wsave;
            }
            fence_proxy_async_smem();                  // the unit is complete: the bulk store after the next __syncwarp
        }
        // ---- (3) trailing update on the tensor cores; the window slides by one block ----
        double af[4][2], bf[4][2];
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            const double dk = __shfl_sync(FULL, dsave, 4 * ks + q);
#pragma unroll
            for (int I = 0; I < 4; ++I) {
                bf[I][ks] = ho.vb[(8 * I + gq) * VBP + 4 * ks + q];
                af[I][ks] = bf[I][ks] * dk;
            }
        }
#pragma unroll
        for (int I = 0; I < 4; ++I)
#pragma unroll
            for (int J = 0; J <= I; ++J) {
                double c[2] = {0.0, 0.0};
                if (I < 3) { c[0] = W[blk(I + 1, J + 1)][0]; c[1] = W[blk(I + 1, J + 1)][1]; }
                dmma(c, af[I][0], bf[J][0]);
                dmma(c, af[I][1], bf[J][1]);
                W[blk(I, J)][0] = c[0]; W[blk(I, J)][1] = c[1];
            }
        // rows slide by eight as well
        {
            const double up = __shfl_sync(FULL, gv, (lane + 8) & 31), en = __shfl_sync(FULL, gv2, (lane - 24) & 31);
            gv = (lane < 24) ? up : en;
        }
        __syncwarp();
        SEG(12);
        if (lane == 0) {
            mbar_arrive(&sh.ho_full[ls]);
            tma_store_1d(LTp + (size_t)k0 * LROW, lst, LT_UNIT_DOUBLES * sizeof(double), l2_evict_first_policy());
        }
    }
    if (lane == 0) {            // every unit is in the slab before the sweeps read it back, and the staging is free for Ss
        bulk_wait();
        fence_proxy_async();
    }
    return ok;
}

// ---- warp 1: fill rows G = Y L^-T (lane = separator row), blocked like the chain: the 32 x 32 window of G's updates in
//      DMMA C fragments, panel by forward substitution with the panel's unit-lower block, trailing update
//      G'[:, J] = G[:, J+1] + G_panel L^T and S -= (G_panel w) G_panel^T on the tensor cores; also the separator part of
//      the fused forward substitution  gS -= G (w y) ----
__device__ __noinline__ void factor_fill(IpShared &sh, const double *__restrict__ HBp, double *__restrict__ GTp, double *__restrict__ Zp, const int NA, const double *__restrict__ g, unsigned tick) {
    const int lane = threadIdx.x & 31;
    const int gq = lane >> 2, q = lane & 3;
    const int nunits = (NA + SUB - 1) / SUB;
    double G[4][4][2];
#pragma unroll
    for (int I = 0; I < 4; ++I)
#pragma unroll
        for (int J = 0; J < 4; ++J) { G[I][J][0] = 0.0; G[I][J][1] = 0.0; }
    double gsacc = 0.0;
    double *gb = sh.u.f.gb, *gst = sh.u.f.gt;       // gst: the panel's unit, at its offsets in GT
    for (int t = 0; t < nunits; ++t) {
        const unsigned ht = tick + t, ls = ht % HO_SLOTS;
        const int k0 = t * SUB;
        // ---- column block 0 of the window -> row layout ----
#pragma unroll
        for (int I = 0; I < 4; ++I)
            *reinterpret_cast<double2 *>(&gb[(8 * I + gq) * VBP + 2 * q]) = make_double2(G[I][0][0], G[I][0][1]);
        __syncwarp();
        double gp[8];
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
            const double2 uu = *reinterpret_cast<const double2 *>(&gb[lane * VBP + j]);
            gp[j] = uu.x; gp[j + 1] = uu.y;
        }
        const bool hasY = (k0 < 32) || (k0 + SUB - 1 >= NA - 32);     // Y = M[sep, chain] is nonzero across the wrap and next to the separator
        if (hasY) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int k = k0 + j;
                double yv = 0.0;
                if (k < NA) {
                    if (k <= lane) yv = HBp[(size_t)(NA + lane) * HB_PITCH + (k + 32 - lane)];
                    else if (k >= NA + lane - 32) yv = HBp[(size_t)k * HB_PITCH + (NA + lane - k)];
                }
                gp[j] = yv - gp[j];
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) gp[j] = -gp[j];
        }
        if (lane == 0) bulk_wait_read();               // the previous panel's unit has left the staging buffer
        __syncwarp();
        PROF_T0(tw2);
        mbar_wait_relaxed(&sh.ho_full[ls], (ht / HO_SLOTS) & 1u);
        PROF_ADD1(PROF_W1_WAIT_HO_FULL, tw2);
        const Handoff &ho = sh.u.f.ho[ls];
        // ---- the panel: g_j -= sum_{m<j} g_m L[k0+j][k0+m] ----
#pragma unroll
        for (int m = 0; m < 7; ++m)                 // right-looking: gp[m] is final, the updates of one column are independent
#pragma unroll
            for (int j = m + 1; j < 8; ++j) gp[j] = fma(-gp[m], ho.l11[j * 8 + m], gp[j]);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            gst[j * FROW + lane] = gp[j];
            gsacc = fma(gp[j], ho.w[j] * ho.y[j], gsacc);
        }
        if (lane < 8) {
            const double w = ho.w[lane];
            gst[lane * FROW + 32] = w;
            Zp[k0 + lane] = w * ho.y[lane];            // z of the predictor (the fused forward half)
        }
        fence_proxy_async_smem();                      // the unit is complete: the bulk store after the next __syncwarp
#pragma unroll
        for (int j = 0; j < 8; j += 2) *reinterpret_cast<double2 *>(&gb[lane * VBP + j]) = make_double2(gp[j], gp[j + 1]);
        __syncwarp();
        if (lane == 0) tma_store_1d(GTp + (size_t)k0 * FROW, gst, GT_UNIT_DOUBLES * sizeof(double), l2_evict_first_policy());
        PROF_T0(tw3);
        // ---- trailing update: G'[I][J] = G[I][J+1] + G_panel[I] L[J]^T ----
        double af[4][2], bf[4][2], wq[2];
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
            wq[ks] = ho.w[4 * ks + q];
#pragma unroll
            for (int I = 0; I < 4; ++I) {
                af[I][ks] = gb[(8 * I + gq) * VBP + 4 * ks + q];
                bf[I][ks] = ho.vb[(8 * I + gq) * VBP + 4 * ks + q];
            }
        }
#pragma unroll
        for (int I = 0; I < 4; ++I)
#pragma unroll
            for (int J = 0; J < 4; ++J) {
                double c[2] = {0.0, 0.0};
                if (J < 3) { c[0] = G[I][J + 1][0]; c[1] = G[I][J + 1][1]; }
                dmma(c, af[I][0], bf[J][0]);
                dmma(c, af[I][1], bf[J][1]);
                G[I][J][0] = c[0]; G[I][J][1] = c[1];
            }
        // ---- S += (G_panel w) G_panel^T (lower blocks; subtracted from M[sep, sep] at the end) ----
#pragma unroll
        for (int I = 0; I < 4; ++I) {
            double c2[4][2];
#pragma unroll
            for (int J = 0; J <= I; ++J) {
                const double2 cc = *reinterpret_cast<const double2 *>(&sh.s.c.sfrag[(blk(I, J) * 32 + lane) * 2]);
                c2[J][0] = cc.x; c2[J][1] = cc.y;
            }
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const double a = af[I][ks] * wq[ks];
#pragma unroll
                for (int J = 0; J <= I; ++J) dmma(c2[J], a, af[J][ks]);
            }
#pragma unroll
            for (int J = 0; J <= I; ++J)
                *reinterpret_cast<double2 *>(&sh.s.c.sfrag[(blk(I, J) * 32 + lane) * 2]) = make_double2(c2[J][0], c2[J][1]);
        }
        __syncwarp();
        PROF_ADD1(PROF_W1_UPDATE, tw3);
        if (lane == 0) mbar_arrive(&sh.ho_empty[ls]);
    }
    if (lane == 0) {            // every unit is in the slab before the sweeps read it back, and the staging is free for their ring
        bulk_wait();
        fence_proxy_async();
    }
    sh.gs[lane] = g[NA + lane] - gsacc;
}

// ---- factorisation of M = H + D with the forward substitution of g; returns false on a non-positive pivot.
//      `tick` counts the hand-off units of this CTA so far (slot / parity bookkeeping of the mbarrier rings); the caller
//      advances it by factor_units(n) afterwards. ----
__device__ __forceinline__ unsigned factor_units(int n) { return (unsigned)((n - 32 + SUB - 1) / SUB); }
__device__ __noinline__ bool factor(IpShared &sh, double *slab, const Layout &L, int n, const double *HB, const double *g, unsigned tick) {
    const Factor F = make_factor(slab, L, n, HB);
    const int NA = F.NA;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int e = threadIdx.x; e < 20 * 32; e += IP_THREADS) sh.s.c.sfrag[e] = 0.0;
    fence_proxy_async();        // the band may have been assembled by this kernel (K2b') and the band-row slots were last
    __syncthreads();            // used by the sweeps, both through the generic proxy; the bulk copies are the async proxy
    PROF_T0(tc0);
    if (warp == 0) {
        if (!factor_chain(sh, F.HB, F.DD, F.LT, NA, g, tick)) sh.flag = 1;
        PROF_ADD(PROF_CHAIN, tc0);
    } else {
        factor_fill(sh, F.HB, F.GT, F.Z, NA, g, tick);
        PROF_ADD1(PROF_FILL, tc0);
    }
    PROF_T0(tc1);
    // ---- separator: S = M[sep, sep] + D_S - G D^-1 G^T, LDL^T in place (warp 1) ----
    double sf[20];
    if (warp == 1) {
#pragma unroll
        for (int e = 0; e < 20; ++e) sf[e] = sh.s.c.sfrag[((e >> 1) * 32 + lane) * 2 + (e & 1)];
    }
    // (the separator block of M: 16 entries per thread, all loads in flight before the barrier)
    double sv[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int e = threadIdx.x + i * IP_THREADS;
        const int r = e >> 5, c = e & 31;
        const int lo = min(r, c), dist = abs(r - c);
        sv[i] = F.HB[(size_t)(NA + lo) * HB_PITCH + dist];
        if (r == c) sv[i] += F.DD[NA + r];
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int e = threadIdx.x + i * IP_THREADS;
        sh.s.Ss[(e >> 5) * 33 + (e & 31)] = sv[i];
    }
    __syncthreads();
    if (warp == 1) {
        const int gq = lane >> 2, q = lane & 3;
#pragma unroll
        for (int I = 0; I < 4; ++I)
#pragma unroll
            for (int J = 0; J <= I; ++J) {
                const int bi = (I * (I + 1)) / 2 + J;
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int r = 8 * I + gq, c = 8 * J + 2 * q + e;
                    sh.s.Ss[r * 33 + c] -= sf[2 * bi + e];
                    if (I != J) sh.s.Ss[c * 33 + r] -= sf[2 * bi + e];
                }
            }
        __syncwarp();
        // right-looking LDL^T in place in shared memory, lane = row (the full square is kept up to date, so row k is also
        // column k).  A loop, not 32 unrolled steps on a register row: that version was 51 KB of SASS run once per
        // factorisation (same speed, a quarter of the kernel's instruction footprint).
        bool ok = true;
#pragma unroll 1
        for (int k = 0; k < 32; ++k) {
            const double d = sh.s.Ss[k * 33 + k];
            if (!(d > 0.0)) ok = false;
            const double w = fast_rcp(d);
            const double l = sh.s.Ss[lane * 33 + k] * w;
            if (lane > k) {
#pragma unroll 4
                for (int c = k + 1; c < 32; ++c) sh.s.Ss[lane * 33 + c] = fma(-l, sh.s.Ss[k * 33 + c], sh.s.Ss[lane * 33 + c]);
                sh.s.Ss[lane * 33 + k] = l;
            }
            if (lane == k) sh.wS[k] = w;
            __syncwarp();
        }
        if (!ok) sh.flag = 1;
    }
    __syncthreads();
    PROF_ADD(PROF_SEP_LDLT, tc1);
    return sh.flag == 0;
}

// ---- sweep ring: one warp consumes the 8-column units of a factor stream in order (from unit 0 up, or from the last unit
//      down), streamed HBM -> shared by bulk copies it issues itself; AHEAD units are in flight.  prime() before the loop;
//      per unit i: wait(), refill(i) by lane 0 once every lane is done with the unit (the unit AHEAD further on goes into
//      the slot of unit i - 1), next() with the loop counter: the cursors walk the slots cyclically, no modulo. ----
template <int SLOTS, int BASE, int UNIT_DOUBLES, int WHO>
struct RingT {
    static constexpr int AHEAD = SLOTS - 1;
    IpShared &sh;
    double *buf;
    unsigned phase;
    uint64_t pol;
    const double *rows;        // the unit stream: units 0 .. nunits - 1, taken from unit 0 up or (down) from the last one
    int nunits, last;
    bool down;
    int sl, sn;                // slots of the next unit to consume and of the next refill
    __device__ RingT(IpShared &s, double *b, const double *r, int nu, bool dn)
        : sh(s), buf(b), phase(s.ring_phase[WHO]), pol(l2_evict_first_policy()), rows(r), nunits(nu), last(nu - 1), down(dn), sl(0), sn(AHEAD) {}
    __device__ __forceinline__ int unit(int i) const { return down ? last - i : i; }      // the i-th unit in order
    __device__ __forceinline__ void issue(int u, int slot) {
        const unsigned bytes = (unsigned)(UNIT_DOUBLES * sizeof(double));
        mbar_expect_tx(&sh.ring_full[BASE + slot], bytes);
        tma_load_1d(buf + slot * UNIT_DOUBLES, rows + (size_t)u * UNIT_DOUBLES, bytes, &sh.ring_full[BASE + slot], pol);
    }
    __device__ __forceinline__ void prime() {
        if ((threadIdx.x & 31) == 0) for (int i = 0; i < AHEAD && i < nunits; ++i) issue(unit(i), i);
    }
    __device__ __forceinline__ const double *wait() {
#ifdef MC_PROFILE
        const long long tw = clock64();
#endif
        mbar_wait(&sh.ring_full[BASE + sl], (phase >> sl) & 1u);
#ifdef MC_PROFILE
        if (blockIdx.x == 0 && (threadIdx.x & 31) == 0) atomicAdd(&g_prof[PROF_RING_WAIT_W0 + WHO], (unsigned long long)(clock64() - tw));
#endif
        phase ^= 1u << sl;
        return buf + sl * UNIT_DOUBLES;
    }
    __device__ __forceinline__ void refill(int i) { if (i + AHEAD < nunits) issue(down ? unit(i) - AHEAD : unit(i) + AHEAD, sn); }
    __device__ __forceinline__ void next() {
        sl = (sl == SLOTS - 1) ? 0 : sl + 1;
        sn = (sn == SLOTS - 1) ? 0 : sn + 1;
    }
    __device__ __forceinline__ void close() { sh.ring_phase[WHO] = phase; }
};
using LtRing = RingT<LT_SLOTS, 0, LT_UNIT_DOUBLES, 0>;
using GtRing = RingT<GT_SLOTS, LT_SLOTS, GT_UNIT_DOUBLES, 1>;

// progress counters between the two warps of a sweep (shared memory, CTA scope)
__device__ __forceinline__ void prog_publish(int *p, int v) { asm volatile("st.release.cta.shared.s32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory"); }
__device__ __forceinline__ int prog_read(const int *p) {
    int v;
    asm volatile("ld.acquire.cta.shared.s32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
    return v;
}
// wait until *p >= need (bounded: a protocol error must not hang the device; it is reported like a failed pivot)
template <bool BACKOFF = false>
__device__ __forceinline__ void prog_wait(IpShared &sh, const int *p, int need) {
    for (int spin = 0; spin < (1 << 18); ++spin) {
        if (prog_read(p) >= need) return;
        if (BACKOFF) __nanosleep(MC_RELAXED_BACKOFF_NS);      // warp 1's waits: it is the one with slack in both sweeps
    }
    sh.flag = 1;
}

// forward sweep (warp 0): y = L^-1 g, one panel of eight columns at a time, as mat-vecs on the tensor cores.  With the
// panel stored as [Q - I; L21] (Q = L11^-1, L21 the 32 rows below) the step is
//   y1 = a1 + (Q - I) a1,   a[k0+8 .. k0+39] -= L21 y1       (rows k0+32 .. k0+39 enter with g).
// The window a lives in DMMA C fragments (every column of the 8 x 8 tile carries the same vector): lane (gq, q) holds
// a[k0 + 8 I + gq], I = 0..3; B operands (a1, y1 at index 4 h + q) come by shuffle.
// z = w y goes to warp 1 (sweep_sep_rhs runs one unit behind) through the queue sw.q, and to the vector Z for the backward
// half of the solve.
__device__ __noinline__ void sweep_forward(IpShared &sh, double *__restrict__ LTp, double *__restrict__ Zp, const int NA, const double *__restrict__ g) {
    const int lane = threadIdx.x & 31;
    const int gq = lane >> 2, q = lane & 3;
    const int nunits = (NA + SUB - 1) / SUB;
    LtRing R(sh, &sh.u.sw.lt[0][0], LTp, nunits, false);
    R.prime();
    double acc[4];
#pragma unroll
    for (int I = 0; I < 4; ++I) acc[I] = (8 * I + gq < NA) ? g[8 * I + gq] : 0.0;
    double gcur = (32 + lane < NA) ? g[32 + lane] : 0.0;       // g of the rows that enter over the next four panels,
    double gnext = (64 + lane < NA) ? g[64 + lane] : 0.0;      // and the block after it (loaded a block ahead)
    for (int u = 0; u < nunits; ++u, R.next()) {
        const int k0 = u * SUB;
        if (u > 0 && (u & 3) == 0) {
            gcur = gnext;
            const int idx = k0 + 64 + lane;
            gnext = (idx < NA) ? g[idx] : 0.0;
        }
        if ((u & 7) == 0 && u >= 8) prog_wait(sh, &sh.prog[1], u - 8);      // queue slots of units u .. u+7 are free again
        const double *lt = R.wait();
        const double ge = __shfl_sync(FULL, gcur, ((u & 3) << 3) + gq);
        double a[5][2];                                  // A fragments: column 4 h + q of the panel, row 8 I + gq
#pragma unroll
        for (int I = 0; I < 5; ++I) {
            a[I][0] = lt_entry(lt, q, 8 * I + gq);
            a[I][1] = lt_entry(lt, 4 + q, 8 * I + gq);
        }
        const double wl = lt[gq * LROW + 32];                    // w of column k0 + gq
        // y1 = a1 + (Q - I) a1: two independent products
        const double b0 = __shfl_sync(FULL, acc[0], 4 * q), b1 = __shfl_sync(FULL, acc[0], 16 + 4 * q);
        double y0[2] = {acc[0], acc[0]}, y1[2] = {0.0, 0.0};
        dmma(y0, a[0][0], b0);
        dmma(y1, a[0][1], b1);
        const double y = y0[0] + y1[0];
        const double n0 = -__shfl_sync(FULL, y, 4 * q), n1 = -__shfl_sync(FULL, y, 16 + 4 * q);
        double nw[4];
#pragma unroll
        for (int I = 0; I < 4; ++I) {                  // block 0 (rows k0+8 ..) first: it is the next panel's a1
            const double c = (I < 3) ? acc[I + 1] : ge;
            double c0[2] = {c, c}, c1[2] = {0.0, 0.0};
            dmma(c0, a[I + 1][0], n0);
            dmma(c1, a[I + 1][1], n1);
            nw[I] = c0[0] + c1[0];
        }
        if (q == 0) {
            const bool in = (k0 + gq < NA);
            const double z = in ? y * wl : 0.0;
            sh.u.sw.q[(u & (QDEPTH - 1)) * SUB + gq] = z;
            if (in) Zp[k0 + gq] = z;
        }
#pragma unroll
        for (int I = 0; I < 4; ++I) acc[I] = nw[I];
        __syncwarp();
        if (lane == 0) { prog_publish(&sh.prog[0], u + 1); R.refill(u); }
    }
    R.close();
    fence_proxy_async();        // the ring slots, read through the generic proxy, are refilled by the backward sweep's bulk copies
}

// separator part of the forward sweep (warp 1, one unit behind warp 0):  gs = g_S - G z
__device__ __noinline__ void sweep_sep_rhs(IpShared &sh, double *__restrict__ GTp, const int NA, const double *__restrict__ g) {
    const int lane = threadIdx.x & 31;
    const int nunits = (NA + SUB - 1) / SUB;
    GtRing R(sh, &sh.u.sw.gt[0][0], GTp, nunits, false);
    R.prime();
    double s0 = 0.0, s1 = 0.0;
    const double gsl = g[NA + lane];
    for (int u = 0; u < nunits; ++u, R.next()) {
        const double *gt = R.wait() + lane;
        prog_wait<true>(sh, &sh.prog[0], u + 1);
        const double *zq = &sh.u.sw.q[(u & (QDEPTH - 1)) * SUB];       // (padding columns: z = 0, g = 0)
#pragma unroll
        for (int s2 = 0; s2 < SUB; s2 += 2) {
            s0 = fma(gt[s2 * FROW], zq[s2], s0);
            s1 = fma(gt[(s2 + 1) * FROW], zq[s2 + 1], s1);
        }
        __syncwarp();
        if (lane == 0) { prog_publish(&sh.prog[1], u + 1); R.refill(u); }
    }
    R.close();
    sh.gs[lane] = gsl - (s0 + s1);
}

// separator solve and the right-hand side of the backward sweep (warp 1, ahead of warp 0's sweep_backward):
//   x_S = S^-1 gs;   t = (y - G^T x_S) w = z - w G^T x_S, from the last unit down, handed over through the queue sw.q.
// z comes from the vector the forward half wrote (plain loads, one unit ahead: it was written in this launch)
__device__ __noinline__ void sweep_sep_solve(IpShared &sh, double *__restrict__ GTp, const double *Zp, const int NA, double *__restrict__ x) {
    const int lane = threadIdx.x & 31;
    const int nunits = (NA + SUB - 1) / SUB;
    GtRing R(sh, &sh.u.sw.gt[0][0], GTp, nunits, true);
    R.prime();
    double a = sh.gs[lane];
#pragma unroll 4
    for (int k = 0; k < 32; ++k) {
        const double yk = __shfl_sync(FULL, a, k);
        const double l = (lane > k) ? sh.s.Ss[lane * 33 + k] : 0.0;
        a = fma(-l, yk, a);
    }
    a *= sh.wS[lane];
#pragma unroll 4
    for (int k = 31; k >= 0; --k) {
        const double xk = __shfl_sync(FULL, a, k);
        const double l = (lane < k) ? sh.s.Ss[k * 33 + lane] : 0.0;
        a = fma(-l, xk, a);
    }
    x[NA + lane] = a;
    // c_k = sum_r G[r][k] x_S[r]: lane = (column k0 + (lane & 7), quarter lane >> 3 of the separator rows)
    const int kl = lane & 7, qr = lane >> 3;
    double xq[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) xq[i] = __shfl_sync(FULL, a, 8 * qr + i);
    double znext = 0.0;
    if (nunits > 0 && R.unit(0) * SUB + kl < NA) znext = Zp[R.unit(0) * SUB + kl];
    for (int i = 0; i < nunits; ++i, R.next()) {
        const int k = R.unit(i) * SUB + kl;
        const double z = znext;
        if (i + 1 < nunits && R.unit(i + 1) * SUB + kl < NA) znext = Zp[R.unit(i + 1) * SUB + kl];
        if ((i & 7) == 0 && i >= 8) prog_wait<true>(sh, &sh.prog[2], i - 8);      // queue slots of the next eight units are free again
        const double *gt = R.wait() + kl * FROW;      // (pitch 33: scalar loads, on distinct banks)
        double c0 = 0.0, c1 = 0.0;
#pragma unroll
        for (int e = 0; e < 8; e += 2) {
            c0 = fma(gt[8 * qr + e], xq[e], c0);
            c1 = fma(gt[8 * qr + e + 1], xq[e + 1], c1);
        }
        double c = c0 + c1;
        c += __shfl_xor_sync(FULL, c, 8);
        c += __shfl_xor_sync(FULL, c, 16);
        if (qr == 0) sh.u.sw.q[(i & (QDEPTH - 1)) * SUB + kl] = (k < NA) ? fma(-c, gt[32], z) : 0.0;      // (padding rows: t = 0)
        __syncwarp();
        if (lane == 0) { prog_publish(&sh.prog[3], i + 1); R.refill(i); }
    }
    R.close();
}

// backward sweep (warp 0): x = L^-T t, one panel at a time from the last one, as mat-vecs on the tensor cores:
//   u = t1 - L21^T x[k0+8 .. k0+39],   x[k0 .. k0+7] = u + (Q - I)^T u.
// The 32 x's below the panel are kept NEGATED as B operands (lane (gq, q): -x[k0 + 8 + 4 i + q], i = 0..7); u and the eight new
// x's come out in C layout (lane (gq, .): row k0 + gq) and move over by shuffle.  Only the two products with the previous
// panel's x and the two with u are on the chain from panel to panel; the other six are issued ahead of them.
// t comes from warp 1 (sweep_sep_solve, running ahead) through the queue sw.q.
__device__ __noinline__ void sweep_backward(IpShared &sh, double *__restrict__ LTp, const int NA, double *__restrict__ x) {
    const int lane = threadIdx.x & 31;
    const int gq = lane >> 2, q = lane & 3;
    const int nunits = (NA + SUB - 1) / SUB;
    LtRing R(sh, &sh.u.sw.lt[0][0], LTp, nunits, true);
    R.prime();
    double nbx[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) nbx[i] = 0.0;
    for (int i = 0; i < nunits; ++i, R.next()) {
        const int k0 = R.unit(i) * SUB;
        const double *lt = R.wait();
        double a[10];                                    // A fragments: column gq of the panel, row 4 c + q
#pragma unroll
        for (int c = 0; c < 10; ++c) a[c] = lt_entry(lt, gq, 4 * c + q);
        double c0[2] = {0.0, 0.0}, c1[2] = {0.0, 0.0};
#pragma unroll
        for (int e = 2; e < 8; e += 2) {
            dmma(c0, a[2 + e], nbx[e]);
            dmma(c1, a[3 + e], nbx[e + 1]);
        }
        dmma(c0, a[2], nbx[0]);
        dmma(c1, a[3], nbx[1]);
        prog_wait(sh, &sh.prog[3], i + 1);
        const double t1 = sh.u.sw.q[(i & (QDEPTH - 1)) * SUB + gq];
        const double uu = t1 + (c0[0] + c1[0]);
        const double u0 = __shfl_sync(FULL, uu, 4 * q), u1 = __shfl_sync(FULL, uu, 16 + 4 * q);
        double d0[2] = {uu, uu}, d1[2] = {0.0, 0.0};
        dmma(d0, a[0], u0);
        dmma(d1, a[1], u1);
        const double x1 = d0[0] + d1[0];
        if (q == 0 && k0 + gq < NA) x[k0 + gq] = x1;
#pragma unroll
        for (int e = 7; e >= 2; --e) nbx[e] = nbx[e - 2];
        nbx[0] = -__shfl_sync(FULL, x1, 4 * q);
        nbx[1] = -__shfl_sync(FULL, x1, 16 + 4 * q);
        __syncwarp();
        if (lane == 0) { prog_publish(&sh.prog[2], i + 1); R.refill(i); }
    }
    R.close();
}

// x = M^-1 g with the stored factor.  fused: the forward part was done inside factor() (predictor).  Both halves run on the
// two warps concurrently: warp 1's separator reduction trails warp 0's forward sweep, then (after the separator solve)
// warp 1's right-hand side t runs ahead of warp 0's backward sweep.
__device__ __noinline__ void solve(IpShared &sh, double *slab, const Layout &L, int n, const double *g, double *x, bool fused) {
    const Factor F = make_factor(slab, L, n, nullptr);      // (the sweeps read the stored factor only)
    const int warp = threadIdx.x >> 5;
    if (threadIdx.x < 4) sh.prog[threadIdx.x] = 0;
    fence_proxy_async();        // the ring area was last accessed through the generic proxy (factor hand-off buffers)
    __syncthreads();
    if (!fused) {
        PROF_T0(t0);
        if (warp == 0) sweep_forward(sh, F.LT, F.Z, F.NA, g);
        else sweep_sep_rhs(sh, F.GT, F.NA, g);
        __syncthreads();
        PROF_ADD1(PROF_FWD_SWEEPS, t0);
    }
    PROF_T0(t3);
    if (warp == 1) sweep_sep_solve(sh, F.GT, F.Z, F.NA, x);
    else sweep_backward(sh, F.LT, F.NA, x);
    __syncthreads();
    PROF_ADD1(PROF_BWD_SWEEPS, t3);
}

// banded cyclic mat-vec out = H v (real-indexed)
__device__ void band_matvec(const double *__restrict__ HB, const double *__restrict__ v, double *__restrict__ out, int n) {
    for (int i = threadIdx.x; i < n; i += IP_THREADS) {
        const double *row = HB + (size_t)i * HB_PITCH;
        double s = row[0] * v[i];
        int j = i;
        for (int k = 1; k <= HBW; ++k) {
            j = (j + 1 == n) ? 0 : j + 1;
            s = fma(row[k], v[j], s);
        }
        j = i;
        for (int k = 1; k <= HBW; ++k) {
            j = (j == 0) ? n - 1 : j - 1;
            s = fma(HB[(size_t)j * HB_PITCH + k], v[j], s);
        }
        out[i] = s;
    }
}

// the CTA's state in dynamic shared memory, its mbarriers initialised
__device__ __forceinline__ IpShared &ip_init_shared() {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    IpShared &sh = *reinterpret_cast<IpShared *>(smem_raw);
    if (threadIdx.x == 0) {
        for (int i = 0; i < HB_SLOTS; ++i) mbar_init(&sh.hb_full[i], 1);
        for (int i = 0; i < HO_SLOTS; ++i) { mbar_init(&sh.ho_full[i], 1); mbar_init(&sh.ho_empty[i], 1); }
        for (int i = 0; i < RING_UNITS; ++i) mbar_init(&sh.ring_full[i], 1);
        sh.ring_phase[0] = 0; sh.ring_phase[1] = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    return sh;
}

// the next instance for this CTA: handed out dynamically (iteration counts differ between instances)
__device__ __forceinline__ int next_instance(IpShared &sh, int *work_counter) {
    __syncthreads();
    if (threadIdx.x == 0) sh.next = atomicAdd(work_counter, 1);
    __syncthreads();
    return sh.next;
}

// ---- sliced schedule of the box phase (DESIGN.md section 3.3), one launch: every instance first runs for at most
//      `slice` iterations; an instance that has not stopped by then is PARKED: its scalars go to its slab (the V_PARK
//      vector), it gets a bucket = its predicted remaining work, and its index is appended to that bucket.  Once no
//      instance is left unstarted, a CTA takes the parked ones from the fullest bucket down (greedy longest-first), so that
//      the launch's tail holds short remainders instead of whole instances.  No CTA waits for another: a CTA parks before
//      it looks for work and leaves only when every bucket is empty, so whatever is parked is taken by a running CTA.
//      Only the order of the work changes: each instance runs the same iterations. ----
constexpr int V_PARK = V_VV;           // the curvature-row phase's scratch vector: free while the box phase runs
enum ParkSlot {                        // doubles of V_PARK
    PARK_MU = 0, PARK_MU0 = 1, PARK_RDTOL = 2, PARK_IT = 3,     // the iteration's state besides the slab vectors
    PARK_TRACE = 8,                    // -DMC_TAIL_TRACE: [start, end] of the first part and of the resumed part
                                       //   (%globaltimer), iterations, SM of the first part, iteration count at parking,
                                       //   predicted remaining iterations
    PARK_MU_HIST = 16,                 // -DMC_TAIL_TRACE: mu after iteration 1, 2, ...
    PARK_LIST = 64                     // ints: entry k of slab r = 1 + the r-th instance parked in bucket k (0: not yet)
};
constexpr int PARK_BUCKETS = 24;
// the ints behind the slabs (SCHED_INTS of them, zeroed before the launch): the work counter, per bucket the instances
// parked in it and the instances taken from it
enum SchedSlot { SCHED_WORK = 0, SCHED_COUNT = 8, SCHED_TAKEN = 40 };
static_assert(SCHED_WORK < SCHED_COUNT && SCHED_COUNT + PARK_BUCKETS <= SCHED_TAKEN && SCHED_TAKEN + PARK_BUCKETS <= SCHED_INTS,
              "the schedule's counters behind the slabs");
static_assert(PARK_MU_HIST + 40 <= PARK_LIST && PARK_LIST + PARK_BUCKETS / 2 <= N_MIN + 64, "V_PARK slots within a vector");

__device__ __forceinline__ double *park_slots(double *ws, const Layout &L, int b) { return vec(ws + (size_t)b * L.stride, L, V_PARK); }
__device__ __forceinline__ int *park_list(double *ws, const Layout &L, int r) { return reinterpret_cast<int *>(park_slots(ws, L, r) + PARK_LIST); }
__device__ __forceinline__ int ld_relaxed(const int *p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// bucket of a parked instance: its predicted remaining iterations, from the rate of mu over the last iteration,
//   r = ceil(log(target / mu) / log(mu / mu_prev)) + 1  clipped to [1, left],
// times its size relative to n_max (ragged batches)
__device__ __forceinline__ int park_bucket(double mu, double mu_prev, double target, int left, int n, int n_max) {
    double r = left;
    if (mu <= target) r = 1.0;
    else if (mu < mu_prev) r = ceil(log(target / mu) / log(mu / mu_prev)) + 1.0;
    r = fmin(fmax(r, 1.0), (double)left);
    return min(PARK_BUCKETS - 1, (int)ceil(r * n / n_max));
}

// thread 0, after the whole CTA's stores of the instance's vectors (a barrier before): park instance b in bucket k
__device__ __forceinline__ void park(int *sched, double *ws, const Layout &L, int b, int k) {
    __threadfence();                                   // the slab and the scalars before the entry that publishes them
    const int r = atomicAdd(&sched[SCHED_COUNT + k], 1);
    atomicExch(&park_list(ws, L, r)[k], b + 1);
}

// the next work item of this CTA: an unstarted instance while there are any, then a parked one from the fullest bucket
// down (sh.flag_resume = 1); B when there is neither
__device__ __forceinline__ int next_work(IpShared &sh, int *sched, double *ws, const Layout &L, int B) {
    __syncthreads();
    if (threadIdx.x == 0) {
        int b = B, resumed = 0;
        if (ld_relaxed(&sched[SCHED_WORK]) < B) b = atomicAdd(&sched[SCHED_WORK], 1);
        if (b >= B) {
            b = B;
            for (int k = PARK_BUCKETS - 1; k >= 0 && !resumed; --k) {
                int t = ld_relaxed(&sched[SCHED_TAKEN + k]);
                while (t < ld_relaxed(&sched[SCHED_COUNT + k])) {      // (counts only grow: entry t exists or is coming)
                    const int seen = atomicCAS(&sched[SCHED_TAKEN + k], t, t + 1);
                    if (seen != t) { t = seen; continue; }
                    // the parking CTA increments the count and then writes the entry, with no wait in between
                    const int *e = &park_list(ws, L, t)[k];
                    int v = 0;
                    for (int spin = 0; spin < (1 << 24) && (v = ld_relaxed(e)) == 0; ++spin) __nanosleep(64);
                    __threadfence();
                    if (v > 0) { b = v - 1; resumed = 1; }
                    break;
                }
            }
        }
        sh.next = b;
        sh.resumed = resumed;
    }
    __syncthreads();
    return sh.next;
}

#ifdef MC_TAIL_TRACE
__device__ __forceinline__ double trace_clock() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return __longlong_as_double((long long)t);
}
#endif

// alpha, status and the iteration count of instance b (the curvature-row phase adds its iterations to the box phase's)
template <bool ADD_ITERS>
__device__ __forceinline__ void write_instance(double *aout, int n, int n_max, const double *AL, int b, int result, int it,
                                               int32_t *status, int32_t *iters_out) {
    __syncthreads();
    for (int i = threadIdx.x; i < n_max; i += IP_THREADS) aout[i] = (i < n) ? AL[i] : 0.0;
    if (threadIdx.x == 0) {
        status[b] = result;
        if (iters_out) iters_out[b] = ADD_ITERS ? iters_out[b] + it : it;
    }
}

// ---- Mehrotra's scalar steps: the affine step length min(1, 1 / max-ratio); the centring target sigma mu with
//      sigma = (mu_aff / mu)^3, mu_aff = the complementarity after the affine step, a polynomial in (ap, ad), over m products;
//      the damped step length min(1, eta / max-ratio) ----
__device__ __forceinline__ double affine_step(double r) { return (r > 1.0) ? 1.0 / r : 1.0; }
__device__ __forceinline__ double centring(double c00, double c01, double c10, double c11, double ap, double ad, double mu, double m) {
    const double sigma = (c00 + ad * c01 + ap * c10 + ap * ad * c11) / m / mu;
    return sigma * sigma * sigma * mu;
}
__device__ __forceinline__ double damped_step(double eta, double r) { return (eta < r) ? eta / r : 1.0; }
// the corrector's complementarity terms tu = sigma mu - s_u l_u + dx dl_u, tl = sigma mu - s_l l_l - dx dl_l of the affine
// direction dx (isu = 1 / s_u, isl = 1 / s_l).  Recomputed by every pass that needs them rather than stored: the same
// expression on the same inputs gives the same bits in each of them.
__device__ __forceinline__ void corrector_terms(double smu, double su, double sl, double lu, double ll, double dx, double isu,
                                                double isl, double &tu, double &tl) {
    const double dlu = lu * (dx * isu - 1.0), dll = -ll * (1.0 + dx * isl);
    tu = smu - su * lu + dx * dlu;
    tl = smu - sl * ll - dx * dll;
}

// slice == 0: every instance runs to the end.  slice > 0: the sliced schedule (instances parked after `slice` iterations,
// resumed longest first).  sched: the SCHED_INTS counters behind the slabs, zeroed before the launch, and (slice > 0) the
// PARK_LIST entries of every slab zeroed too.
__global__ void __launch_bounds__(IP_THREADS, 8)
mincurv_pdip_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, double *__restrict__ ws, Layout L,
                    PdipParams prm, int slice, double *__restrict__ alpha_out, int32_t *__restrict__ status,
                    int32_t *__restrict__ iters_out, int *__restrict__ sched) {
#ifdef MC_DEBUG_SM_LIMIT       // contention experiments: only the first MC_DEBUG_SM_LIMIT SMs take work (full occupancy on those)
    {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        if (smid >= MC_DEBUG_SM_LIMIT) return;
    }
#endif
    IpShared &sh = ip_init_shared();
    unsigned tick = 0;      // hand-off units of the factorisations so far (uniform across the CTA)
    for (int b; (b = next_work(sh, sched, ws, L, B)) < B;) {
        const bool resume = sh.resumed;
        const int n = n_pts ? n_pts[b] : n_max;
        double *aout = alpha_out + (size_t)b * n_max;
        if (!resume && status[b] != 0) {
            for (int i = threadIdx.x; i < n_max; i += IP_THREADS) aout[i] = 0.0;
            if (iters_out && threadIdx.x == 0) iters_out[b] = 0;
            continue;
        }
        PROF_T0(tq0);
#ifdef MC_TAIL_TRACE
        if (threadIdx.x == 0) {
            double *PK = park_slots(ws, L, b);
            if (!resume) {
                unsigned smid;
                asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
                PK[PARK_TRACE + 2] = 0.0; PK[PARK_TRACE + 3] = 0.0; PK[PARK_TRACE + 5] = smid;
                PK[PARK_TRACE + 6] = 0.0; PK[PARK_TRACE + 7] = 0.0;
            }
            PK[PARK_TRACE + (resume ? 2 : 0)] = trace_clock();
        }
#endif
        double *slab = ws + (size_t)b * L.stride;
        const double *HB = ws + (size_t)*band_owner(slab, L) * L.stride + L.o_hb;      // (shared centre lines: the owner's)
        const double *__restrict__ LB = vec(slab, L, V_LB), *__restrict__ UB = vec(slab, L, V_UB), *__restrict__ F = vec(slab, L, V_F);
        double *__restrict__ AL = vec(slab, L, V_ALPHA), *__restrict__ LU = vec(slab, L, V_LU), *__restrict__ LL = vec(slab, L, V_LL), *__restrict__ RD = vec(slab, L, V_RD);
        double *__restrict__ RHS = vec(slab, L, V_RHS), *__restrict__ DX = vec(slab, L, V_DX), *__restrict__ DXA = vec(slab, L, V_DXA);
        double *__restrict__ DD = vec(slab, L, V_DD), *__restrict__ SU = vec(slab, L, V_SU), *__restrict__ SL = vec(slab, L, V_SL);
        double *G0 = vec(slab, L, V_T0);
        if (threadIdx.x == 0) sh.flag = 0;
        double mu0, rd_tol, mu;
        int it;
        if (resume) {                  // a parked instance: its vectors are in the slab, its scalars in V_PARK
            const double *PK = park_slots(ws, L, b);
            mu = PK[PARK_MU]; mu0 = PK[PARK_MU0]; rd_tol = PK[PARK_RDTOL]; it = (int)PK[PARK_IT];
        } else {
            // ---------------- initial point: box centre, multipliers from the gradient ----------------
            for (int i = threadIdx.x; i < n; i += IP_THREADS) AL[i] = 0.5 * (LB[i] + UB[i]);
            __syncthreads();
            band_matvec(HB, AL, G0, n);
            __syncthreads();
            double gmax = 0.0, fmaxv = 0.0;
#pragma unroll 1
            for (int i = threadIdx.x; i < n; i += IP_THREADS) {
                const double gi = G0[i] + F[i];
                G0[i] = gi;
                gmax = fmax(gmax, fabs(gi));
                fmaxv = fmax(fmaxv, fabs(F[i]));
            }
            gmax = block_reduce<1>(gmax, sh.red);
            fmaxv = block_reduce<1>(fmaxv, sh.red);
            const double lam0 = prm.lam0_rel * gmax + 1e-300;
            double musum = 0.0;
#pragma unroll 1
            for (int i = threadIdx.x; i < n; i += IP_THREADS) {
                const double gi = G0[i];
                const double lu = fmax(-gi, 0.0) + lam0, ll = fmax(gi, 0.0) + lam0;
                const double rd = gi + lu - ll;
                LU[i] = lu; LL[i] = ll;
                RD[i] = rd;
                const double a = AL[i];
                // slacks are carried as variables of their own: recomputing ub - alpha loses them to
                // cancellation once s << eps |alpha| (late iterations), see DESIGN.md
                const double su = UB[i] - a, sl = a - LB[i];
                const double isu = 1.0 / su, isl = 1.0 / sl;
                SU[i] = su; SL[i] = sl;
                DD[i] = lu * isu + ll * isl; RHS[i] = -rd + lu - ll;       // barrier diagonal, affine right-hand side
                musum += su * lu + sl * ll;
            }
            musum = block_reduce<0>(musum, sh.red);
            mu0 = musum / (2.0 * n);
            rd_tol = prm.rd_rel * (fmaxv + gmax) + 1e-300;
            mu = mu0;
            it = 0;
        }
        int result = -1;               // still running
        const int it_end = (slice > 0 && !resume) ? min(slice, prm.max_iter) : prm.max_iter;

        // Vector phases: the state of an iteration is alpha, s_u, s_l, l_u, l_l, r_d (AL SU SL LU LL RD) and the next
        // factorisation's DD and RHS; within it the affine direction DXA and the combined one DX.  Everything else is
        // recomputed where it is used, which costs less than its memory traffic: the reciprocals 1/s_u, 1/s_l (IEEE
        // divisions: the same bits in every pass) and the corrector terms tu, tl (corrector_terms).  Step lengths come
        // from max-ratios.  RHS carries the corrector's right-hand side from its pass to the update pass.
        // Every thread owns the elements i = tid + k * 64; the loops take them in groups of VG with all loads of a
        // group issued before the first use (the vectors live in L2/HBM: one element at a time, each trip of a loop
        // paid the full memory latency).
        // The barrier diagonal DD = lu / su + ll / sl and the affine right-hand side RHS = -rd + lu - ll of an iteration
        // are computed where their inputs are: by the loop above for the first iteration, by the update pass of the
        // previous iteration for the others.  A parked instance resumes from the state alone.
        constexpr int VG = 4, VS = VG * IP_THREADS;
        for (; it < it_end; ++it) {
            PROF_T0(tf0);
            const bool fok = factor(sh, slab, L, n, HB, RHS, tick);
            tick += factor_units(n);
            if (!fok) { result = 3; break; }
            PROF_ADD(PROF_FACTOR, tf0);
            PROF_T0(ts0);
            solve(sh, slab, L, n, RHS, DXA, true);
            PROF_ADD(PROF_SOLVE_PRED, ts0);
            // ---- affine direction: step lengths 1 / max-ratio; mu_aff as a polynomial in (ap, ad) ----
            PROF_T0(tv2);
            double rp = 0.0, rdl = 0.0, c00 = 0.0, c01 = 0.0, c10 = 0.0, c11 = 0.0;
#pragma unroll 1
            for (int i0 = threadIdx.x; i0 < n; i0 += VS) {
                double su[VG], sl[VG], lu[VG], ll[VG], dx[VG];
#pragma unroll
                for (int k = 0; k < VG; ++k) {
                    const int i = min(i0 + k * IP_THREADS, n - 1);
                    su[k] = SU[i]; sl[k] = SL[i]; lu[k] = LU[i]; ll[k] = LL[i]; dx[k] = DXA[i];
                }
#pragma unroll
                for (int k = 0; k < VG; ++k) {
                    if (i0 + k * IP_THREADS < n) {
                        const double isu = 1.0 / su[k], isl = 1.0 / sl[k];
                        const double p = dx[k] * isu, m = dx[k] * isl;
                        rp = fmax(rp, fmax(p, -m));                 // s_u - a dx >= 0, s_l + a dx >= 0
                        rdl = fmax(rdl, fmax(1.0 - p, 1.0 + m));    // dlu / lu = -1 + p, dll / ll = -1 - m
                        const double dlu = lu[k] * (p - 1.0), dll = -ll[k] * (1.0 + m);
                        c00 += su[k] * lu[k] + sl[k] * ll[k];
                        c01 += su[k] * dlu + sl[k] * dll;           // coefficient of ad
                        c10 += dx[k] * (ll[k] - lu[k]);             // coefficient of ap
                        c11 += dx[k] * (dll - dlu);                 // coefficient of ap * ad
                    }
                }
            }
            rp = block_reduce<1>(rp, sh.red);
            rdl = block_reduce<1>(rdl, sh.red);
            double ap = affine_step(rp), ad = affine_step(rdl);
            c00 = block_reduce<0>(c00, sh.red); c01 = block_reduce<0>(c01, sh.red);
            c10 = block_reduce<0>(c10, sh.red); c11 = block_reduce<0>(c11, sh.red);
            const double smu = centring(c00, c01, c10, c11, ap, ad, mu, 2.0 * n);
            PROF_ADD(PROF_AFFINE, tv2);
            PROF_T0(tv3);
            // ---- corrector right-hand side ----
#pragma unroll 1
            for (int i0 = threadIdx.x; i0 < n; i0 += VS) {
                double su[VG], sl[VG], lu[VG], ll[VG], dx[VG], rd[VG];
#pragma unroll
                for (int k = 0; k < VG; ++k) {
                    const int i = min(i0 + k * IP_THREADS, n - 1);
                    su[k] = SU[i]; sl[k] = SL[i]; lu[k] = LU[i]; ll[k] = LL[i]; dx[k] = DXA[i]; rd[k] = RD[i];
                }
#pragma unroll
                for (int k = 0; k < VG; ++k) {
                    const int i = i0 + k * IP_THREADS;
                    if (i < n) {
                        const double isu = 1.0 / su[k], isl = 1.0 / sl[k];
                        double tu, tl;
                        corrector_terms(smu, su[k], sl[k], lu[k], ll[k], dx[k], isu, isl, tu, tl);
                        RHS[i] = -rd[k] - tu * isu + tl * isl;
                    }
                }
            }
            __syncthreads();
            PROF_ADD(PROF_CORR_RHS, tv3);
            PROF_T0(ts1);
            solve(sh, slab, L, n, RHS, DX, false);
            PROF_ADD(PROF_SOLVE_CORR, ts1);
            PROF_T0(tv4);
            rp = 0.0; rdl = 0.0;
#pragma unroll 1
            for (int i0 = threadIdx.x; i0 < n; i0 += VS) {
                double su[VG], sl[VG], lu[VG], ll[VG], dxa[VG], dx[VG];
#pragma unroll
                for (int k = 0; k < VG; ++k) {
                    const int i = min(i0 + k * IP_THREADS, n - 1);
                    su[k] = SU[i]; sl[k] = SL[i]; lu[k] = LU[i]; ll[k] = LL[i]; dxa[k] = DXA[i]; dx[k] = DX[i];
                }
#pragma unroll
                for (int k = 0; k < VG; ++k) {
                    if (i0 + k * IP_THREADS < n) {
                        const double isu = 1.0 / su[k], isl = 1.0 / sl[k];
                        double tu, tl;
                        corrector_terms(smu, su[k], sl[k], lu[k], ll[k], dxa[k], isu, isl, tu, tl);
                        const double dlu = (tu + lu[k] * dx[k]) * isu, dll = (tl - ll[k] * dx[k]) * isl;
                        rp = fmax(rp, fmax(dx[k] * isu, -dx[k] * isl));
                        rdl = fmax(rdl, fmax(-dlu / lu[k], -dll / ll[k]));
                    }
                }
            }
            rp = block_reduce<1>(rp, sh.red);
            rdl = block_reduce<1>(rdl, sh.red);
            ap = damped_step(prm.eta, rp);
            ad = damped_step(prm.eta, rdl);
            PROF_ADD(PROF_STEPLEN, tv4);
            PROF_T0(tv5);
            double musum2 = 0.0, rdmax = 0.0, dxmax = 0.0, amax = 0.0;
            constexpr int VG2 = 2, VS2 = VG2 * IP_THREADS;        // 10 input vectors: groups of two
#pragma unroll 1
            for (int i0 = threadIdx.x; i0 < n; i0 += VS2) {
                double su[VG2], sl[VG2], lu[VG2], ll[VG2], dxa[VG2], dx[VG2], al[VG2], rd[VG2], rh[VG2], dd[VG2];
#pragma unroll
                for (int k = 0; k < VG2; ++k) {
                    const int i = min(i0 + k * IP_THREADS, n - 1);
                    su[k] = SU[i]; sl[k] = SL[i]; lu[k] = LU[i]; ll[k] = LL[i]; dxa[k] = DXA[i]; dx[k] = DX[i];
                    al[k] = AL[i]; rd[k] = RD[i]; rh[k] = RHS[i]; dd[k] = DD[i];
                }
#pragma unroll
                for (int k = 0; k < VG2; ++k) {
                    const int i = i0 + k * IP_THREADS;
                    if (i < n) {
                        const double isu = 1.0 / su[k], isl = 1.0 / sl[k];
                        double tu, tl;
                        corrector_terms(smu, su[k], sl[k], lu[k], ll[k], dxa[k], isu, isl, tu, tl);
                        const double dlu = (tu + lu[k] * dx[k]) * isu, dll = (tl - ll[k] * dx[k]) * isl;
                        const double an = al[k] + ap * dx[k], lun = lu[k] + ad * dlu, lln = ll[k] + ad * dll;
                        const double sun = su[k] - ap * dx[k], sln = sl[k] + ap * dx[k];
                        // H dx = rhs - D dx  (M dx = rhs)
                        const double rdn = rd[k] + ap * (rh[k] - dd[k] * dx[k]) + ad * (dlu - dll);
                        const double isun = 1.0 / sun, isln = 1.0 / sln;
                        AL[i] = an; LU[i] = lun; LL[i] = lln; RD[i] = rdn; SU[i] = sun; SL[i] = sln;
                        // the next iteration's barrier diagonal and affine right-hand side (the expressions of the
                        // initial point; unused if this iteration is the last)
                        DD[i] = lun * isun + lln * isln; RHS[i] = -rdn + lun - lln;
                        musum2 += sun * lun + sln * lln;
                        rdmax = fmax(rdmax, fabs(rdn));
                        dxmax = fmax(dxmax, fabs(dx[k]));
                        amax = fmax(amax, fabs(an));
                    }
                }
            }
            if (threadIdx.x == 0) park_slots(ws, L, b)[PARK_MU] = mu;      // mu before this iteration (read when parking)
            mu = block_reduce<0>(musum2, sh.red) / (2.0 * n);
            rdmax = block_reduce<1>(rdmax, sh.red);
            PROF_ADD(PROF_UPDATE, tv5);
#ifdef MC_TAIL_TRACE
            if (threadIdx.x == 0 && it < PARK_LIST - PARK_MU_HIST) {
                park_slots(ws, L, b)[PARK_MU_HIST + it] = mu;
                park_slots(ws, L, b)[PARK_MU0] = mu0;
            }
#endif
            // weakly active bounds converge like sqrt(mu): also require that the step itself has become small
            bool settled = true;
            if (prm.dx_rel > 0.0 && mu <= prm.mu_rel * mu0) {
                dxmax = block_reduce<1>(dxmax, sh.red);
                amax = block_reduce<1>(amax, sh.red);
                settled = ap * dxmax <= prm.dx_rel * fmax(amax, 0.01);
            }
            if (mu <= prm.mu_rel * mu0 && rdmax <= rd_tol && settled) { result = 0; ++it; break; }
            if (mu <= 1e-4 * prm.mu_rel * mu0) { result = (rdmax <= 1e3 * rd_tol) ? 0 : 2; ++it; break; }   // complementarity exhausted
        }
        if (result < 0 && it < prm.max_iter) {        // the slice is over: park the instance
            if (threadIdx.x == 0) {
                double *PK = park_slots(ws, L, b);
                const double mu_prev = PK[PARK_MU];     // the rate of the last iteration predicts the remaining ones
                PK[PARK_MU] = mu; PK[PARK_MU0] = mu0; PK[PARK_RDTOL] = rd_tol; PK[PARK_IT] = it;
#ifdef MC_TAIL_TRACE
                PK[PARK_TRACE + 1] = trace_clock();
                PK[PARK_TRACE + 6] = it;
                PK[PARK_TRACE + 7] = park_bucket(mu, mu_prev, prm.mu_rel * mu0, prm.max_iter - it, n, n);
#endif
                park(sched, ws, L, b, park_bucket(mu, mu_prev, prm.mu_rel * mu0, prm.max_iter - it, n, n_max));
            }
            continue;
        }
        if (result < 0) result = 2;                    // iteration cap
        write_instance<false>(aout, n, n_max, AL, b, result, it, status, iters_out);
#ifdef MC_TAIL_TRACE
        if (threadIdx.x == 0) {
            double *PK = park_slots(ws, L, b);
            PK[PARK_TRACE + (resume ? 3 : 1)] = trace_clock();
            PK[PARK_TRACE + 4] = it;
        }
#endif
        PROF_ADD(PROF_TOTAL, tq0);
#ifdef MC_PROFILE
        if (blockIdx.x == 0 && threadIdx.x == 0) { atomicAdd(&g_prof[PROF_NQP], 1ull); atomicAdd(&g_prof[PROF_ITERS], (unsigned long long)it); }
#endif
    }
}

// resident CTAs per SM of a solver kernel on the current device (registers and shared memory both count)
template <typename K>
static int ctas_per_sm(K kernel) {
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernel, IP_THREADS, sizeof(IpShared)) != cudaSuccess) return 1;
    return nb > 0 ? nb : 1;
}

// launch shape of a persistent solver kernel: per_sm resident CTAs on every SM, but no more CTAs than instances; the counter
// that hands out the instances sits behind the slabs
struct SolverGrid {
    int grid;
    int *counter;
};
static SolverGrid solver_grid(int B, int n_max, void *workspace, int per_sm) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int grid = sms * (per_sm > 0 ? per_sm : 1);
    if (grid > B) grid = B;
    return {grid, (int *)((char *)workspace + mincurv_slabs_bytes(B, n_max))};
}

// launches a solver kernel (CTA state in dynamic shared memory); its work counter, if it has one, starts from zero
template <typename... P, typename... A>
static int launch_solver(void (*kernel)(P...), int grid, int *work_counter, cudaStream_t stream, A... args) {
    // (per launch: the attribute is per device and a process may drive several)
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(IpShared));
    if (e != cudaSuccess) return (int)e;
    if (work_counter) cudaMemsetAsync(work_counter, 0, sizeof(int), stream);
    kernel<<<grid, IP_THREADS, sizeof(IpShared), stream>>>(args...);
    return 0;
}

// ================================================================================================
// K2b' -- the full QP of tph.opt_min_curv including the curvature rows |k_ref + E a| <= kappa_bound, for the
// instances whose box-only optimum violates them (status 4 after K2c).  Same Mehrotra iteration; the rows enter
// with slacks s3, s4 (infeasible start allowed) and multipliers l3, l4:
//   M = H + D_box + E^T W E = E^T (I + W) E + D_box,  W = l3/s3 + l4/s4      -> weighted band assembly per iteration
//   rhs = -(f + lu - ll) - tu/su + tl/sl - E^T v,  v = (kl - k_ref) + l3 - l4 + (t3 + l3 rp3)/s3 - (t4 + l4 rp4)/s4
// with kl = k_ref + E a carried incrementally and E, E^T applied in O(N) operator form (mincurv_ops.cuh).
// PROX: the Hessian is H + prox_mu I (the projection QP of mc_mincurv_solve_batch_ex, whose prox stage put prox_mu on the
// band's diagonal and its linear term in V_F for the box phase): + prox_mu a in the gradient and the residuals, + prox_mu
// on the factored diagonal.  Without PROX prox_mu is not read.
// kb_batch [B] or NULL: the bound of each instance's rows (NULL: kb for all).  A flagged instance whose bound is not finite
// or not > 0 is refused with status -1 (the finalize stage refuses it before it could be flagged).
// ================================================================================================
template <bool PROX>
__global__ void __launch_bounds__(IP_THREADS, 8)
mincurv_pdip_kappa_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, double *__restrict__ ws, Layout L,
                          PdipParams prm, double kb_scalar, double *__restrict__ alpha_out, int32_t *__restrict__ status,
                          int32_t *__restrict__ iters_out, int *__restrict__ work_counter, double prox_mu,
                          const double *__restrict__ kb_batch) {
    IpShared &sh = ip_init_shared();
    unsigned tick = 0;
    for (int b; (b = next_instance(sh, work_counter)) < B;) {
        if (status[b] != 4) continue;
        const double kb = kb_batch ? kb_batch[b] : kb_scalar;
        if (!(kb > 0.0 && kb < INFINITY)) {     // (a thread that reads the -1 already leaves above: both go on to the
            if (threadIdx.x == 0) status[b] = -1;   //  next instance's barrier)
            continue;
        }
        const int n = n_pts ? n_pts[b] : n_max;
        double *aout = alpha_out + (size_t)b * n_max;
        double *slab = ws + (size_t)b * L.stride;
        const double *__restrict__ LB = vec(slab, L, V_LB), *__restrict__ UB = vec(slab, L, V_UB), *__restrict__ F = vec(slab, L, V_F);
        const double *__restrict__ KR = vec(slab, L, V_KREF);
        double *__restrict__ AL = vec(slab, L, V_ALPHA), *__restrict__ LU = vec(slab, L, V_LU), *__restrict__ LL = vec(slab, L, V_LL);
        double *__restrict__ RHS = vec(slab, L, V_RHS), *__restrict__ DX = vec(slab, L, V_DX), *__restrict__ DD = vec(slab, L, V_DD);
        double *__restrict__ TU = vec(slab, L, V_DLU), *__restrict__ TL = vec(slab, L, V_DLL), *__restrict__ SU = vec(slab, L, V_SU), *__restrict__ SL = vec(slab, L, V_SL);
        double *__restrict__ ISU = vec(slab, L, V_ISU), *__restrict__ ISL = vec(slab, L, V_ISL);
        double *__restrict__ S3 = vec(slab, L, V_S3), *__restrict__ S4 = vec(slab, L, V_S4), *__restrict__ L3 = vec(slab, L, V_L3), *__restrict__ L4 = vec(slab, L, V_L4);
        double *__restrict__ KL = vec(slab, L, V_KL), *__restrict__ WK = vec(slab, L, V_WK), *__restrict__ EDX = vec(slab, L, V_EDX);
        double *__restrict__ T3 = vec(slab, L, V_T3K), *__restrict__ T4 = vec(slab, L, V_T4K), *__restrict__ VV = vec(slab, L, V_VV), *__restrict__ ETV = vec(slab, L, V_RD);
        double *t0 = vec(slab, L, V_T0), *t1 = vec(slab, L, V_T1), *t2 = vec(slab, L, V_T2), *t3 = vec(slab, L, V_T3), *t4 = vec(slab, L, V_T4), *t5 = vec(slab, L, V_T5);
        const double m4 = 4.0 * n;
        if (threadIdx.x == 0) sh.flag = 0;

        // ---- start: box centre; kl = k_ref + E a; gradient g = E^T (E a) + f ----
        for (int i = threadIdx.x; i < n; i += IP_THREADS) AL[i] = 0.5 * (LB[i] + UB[i]);
        __syncthreads();
        apply_E(slab, L, n, AL, EDX, t0, t1, t2, t3, t4, t5);
        apply_Et(slab, L, n, EDX, ETV, t0, t1, t2, t3, t4, t5);
        double gmax = 0.0, fmaxv = 0.0;
        if constexpr (PROX) {
            for (int i = threadIdx.x; i < n; i += IP_THREADS) ETV[i] += prox_mu * AL[i];
        }
        for (int i = threadIdx.x; i < n; i += IP_THREADS) {
            gmax = fmax(gmax, fabs(ETV[i] + F[i]));
            fmaxv = fmax(fmaxv, fabs(F[i]));
        }
        gmax = block_reduce<1>(gmax, sh.red);
        fmaxv = block_reduce<1>(fmaxv, sh.red);
        const double lam0 = prm.lam0_rel * gmax + 1e-300;
        double musum = 0.0;
        for (int i = threadIdx.x; i < n; i += IP_THREADS) {
            const double gi = ETV[i] + F[i];
            const double lu = fmax(-gi, 0.0) + lam0, ll = fmax(gi, 0.0) + lam0;
            const double a = AL[i], su = UB[i] - a, sl = a - LB[i];
            const double kl = KR[i] + EDX[i];
            const double s3 = fmax(kb - kl, 1e-2 * kb), s4 = fmax(kb + kl, 1e-2 * kb);
            LU[i] = lu; LL[i] = ll; SU[i] = su; SL[i] = sl; ISU[i] = 1.0 / su; ISL[i] = 1.0 / sl;
            KL[i] = kl; S3[i] = s3; S4[i] = s4; L3[i] = lam0; L4[i] = lam0;
            musum += su * lu + sl * ll + (s3 + s4) * lam0;
        }
        musum = block_reduce<0>(musum, sh.red);
        const double mu0 = musum / m4;
        const double rd_tol = prm.rd_rel * (fmaxv + gmax) + 1e-300;
        double mu = mu0;
        int it = 0, result = 2;
        double rdmax = 1e300, rpmax = 1e300;
        for (it = 0; it < prm.max_iter + 20; ++it) {
            // ---- weights, barrier diagonal, affine right-hand side ----
            for (int i = threadIdx.x; i < n; i += IP_THREADS) {
                const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i];
                const double rp3 = kl + s3 - kb, rp4 = -kl + s4 - kb;
                WK[i] = l3 / s3 + l4 / s4;
                if constexpr (PROX) DD[i] = LU[i] * ISU[i] + LL[i] * ISL[i] + prox_mu;
                else DD[i] = LU[i] * ISU[i] + LL[i] * ISL[i];
                VV[i] = (kl - KR[i]) + l3 * rp3 / s3 - l4 * rp4 / s4;       // affine: t3 = -s3 l3, t4 = -s4 l4
            }
            __syncthreads();
            assemble_hband(slab, L, n, WK, sh.u.win);     // the tile area is free between the sweeps and the next factorisation
            __syncthreads();
            apply_Et(slab, L, n, VV, ETV, t0, t1, t2, t3, t4, t5);
            if constexpr (PROX) {
                for (int i = threadIdx.x; i < n; i += IP_THREADS) RHS[i] = -F[i] - ETV[i] - prox_mu * AL[i];
            } else {
                for (int i = threadIdx.x; i < n; i += IP_THREADS) RHS[i] = -F[i] - ETV[i];
            }
            __syncthreads();
            const bool fok = factor(sh, slab, L, n, slab + L.o_hb, RHS, tick);      // (the band assembled above, own slab)
            tick += factor_units(n);
            if (!fok) {
                // E^T W E with W = l/s -> 1e12 and beyond is no longer numerically SPD: accept a late iterate, else give up
                result = (mu <= 1e-7 * mu0 && rdmax <= 1e3 * rd_tol && rpmax <= 1e-6 * kb) ? 0 : 3;
                break;
            }
            solve(sh, slab, L, n, RHS, DX, true);
            apply_E(slab, L, n, DX, EDX, t0, t1, t2, t3, t4, t5);
            // ---- affine step lengths and centring ----
            double rp = 0.0, rdl = 0.0, c00 = 0.0, c01 = 0.0, c10 = 0.0, c11 = 0.0;
            for (int i = threadIdx.x; i < n; i += IP_THREADS) {
                const double su = SU[i], sl = SL[i], lu = LU[i], ll = LL[i], dx = DX[i];
                const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i], ed = EDX[i];
                const double p = dx * ISU[i], m = dx * ISL[i];
                const double ds3 = -(kl + s3 - kb) - ed, ds4 = -(-kl + s4 - kb) + ed;
                const double dlu = lu * (p - 1.0), dll = -ll * (1.0 + m);
                const double dl3 = -l3 - l3 * ds3 / s3, dl4 = -l4 - l4 * ds4 / s4;
                rp = fmax(rp, fmax(fmax(p, -m), fmax(-ds3 / s3, -ds4 / s4)));
                rdl = fmax(rdl, fmax(fmax(1.0 - p, 1.0 + m), fmax(-dl3 / l3, -dl4 / l4)));
                c00 += su * lu + sl * ll + s3 * l3 + s4 * l4;
                c01 += su * dlu + sl * dll + s3 * dl3 + s4 * dl4;
                c10 += dx * (ll - lu) + ds3 * l3 + ds4 * l4;
                c11 += dx * (dll - dlu) + ds3 * dl3 + ds4 * dl4;
            }
            rp = block_reduce<1>(rp, sh.red);
            rdl = block_reduce<1>(rdl, sh.red);
            double ap = affine_step(rp), ad = affine_step(rdl);
            c00 = block_reduce<0>(c00, sh.red); c01 = block_reduce<0>(c01, sh.red);
            c10 = block_reduce<0>(c10, sh.red); c11 = block_reduce<0>(c11, sh.red);
            const double smu = centring(c00, c01, c10, c11, ap, ad, mu, m4);
            // ---- corrector right-hand side ----
            for (int i = threadIdx.x; i < n; i += IP_THREADS) {
                const double su = SU[i], sl = SL[i], lu = LU[i], ll = LL[i], dx = DX[i], isu = ISU[i], isl = ISL[i];
                const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i], ed = EDX[i];
                const double rp3 = kl + s3 - kb, rp4 = -kl + s4 - kb;
                const double ds3 = -rp3 - ed, ds4 = -rp4 + ed;
                const double dlu = lu * (dx * isu - 1.0), dll = -ll * (1.0 + dx * isl);
                const double dl3 = -l3 - l3 * ds3 / s3, dl4 = -l4 - l4 * ds4 / s4;
                const double tu = smu - su * lu + dx * dlu, tl = smu - sl * ll - dx * dll;
                const double q3 = smu - s3 * l3 - ds3 * dl3, q4 = smu - s4 * l4 - ds4 * dl4;
                TU[i] = tu; TL[i] = tl; T3[i] = q3; T4[i] = q4;
                VV[i] = (kl - KR[i]) + l3 - l4 + (q3 + l3 * rp3) / s3 - (q4 + l4 * rp4) / s4;
                RHS[i] = -(F[i] + lu - ll) - tu * isu + tl * isl;
            }
            __syncthreads();
            apply_Et(slab, L, n, VV, ETV, t0, t1, t2, t3, t4, t5);
            if constexpr (PROX) {
                for (int i = threadIdx.x; i < n; i += IP_THREADS) RHS[i] -= ETV[i] + prox_mu * AL[i];
            } else {
                for (int i = threadIdx.x; i < n; i += IP_THREADS) RHS[i] -= ETV[i];
            }
            __syncthreads();
            solve(sh, slab, L, n, RHS, DX, false);
            apply_E(slab, L, n, DX, EDX, t0, t1, t2, t3, t4, t5);
            rp = 0.0; rdl = 0.0;
            for (int i = threadIdx.x; i < n; i += IP_THREADS) {
                const double lu = LU[i], ll = LL[i], dx = DX[i], isu = ISU[i], isl = ISL[i];
                const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i], ed = EDX[i];
                const double ds3 = -(kl + s3 - kb) - ed, ds4 = -(-kl + s4 - kb) + ed;
                const double dlu = (TU[i] + lu * dx) * isu, dll = (TL[i] - ll * dx) * isl;
                const double dl3 = (T3[i] - l3 * ds3) / s3, dl4 = (T4[i] - l4 * ds4) / s4;
                rp = fmax(rp, fmax(fmax(dx * isu, -dx * isl), fmax(-ds3 / s3, -ds4 / s4)));
                rdl = fmax(rdl, fmax(fmax(-dlu / lu, -dll / ll), fmax(-dl3 / l3, -dl4 / l4)));
            }
            rp = block_reduce<1>(rp, sh.red);
            rdl = block_reduce<1>(rdl, sh.red);
            ap = damped_step(prm.eta, rp);
            ad = damped_step(prm.eta, rdl);
            double musum2 = 0.0;
            rpmax = 0.0;
            for (int i = threadIdx.x; i < n; i += IP_THREADS) {
                const double su = SU[i], sl = SL[i], lu = LU[i], ll = LL[i], dx = DX[i];
                const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i], ed = EDX[i];
                const double ds3 = -(kl + s3 - kb) - ed, ds4 = -(-kl + s4 - kb) + ed;
                const double dlu = (TU[i] + lu * dx) * ISU[i], dll = (TL[i] - ll * dx) * ISL[i];
                const double dl3 = (T3[i] - l3 * ds3) / s3, dl4 = (T4[i] - l4 * ds4) / s4;
                const double sun = su - ap * dx, sln = sl + ap * dx, s3n = s3 + ap * ds3, s4n = s4 + ap * ds4;
                const double lun = lu + ad * dlu, lln = ll + ad * dll, l3n = l3 + ad * dl3, l4n = l4 + ad * dl4;
                const double kln = kl + ap * ed;
                AL[i] += ap * dx; SU[i] = sun; SL[i] = sln; ISU[i] = 1.0 / sun; ISL[i] = 1.0 / sln;
                LU[i] = lun; LL[i] = lln; S3[i] = s3n; S4[i] = s4n; L3[i] = l3n; L4[i] = l4n; KL[i] = kln;
                VV[i] = (kln - KR[i]) + l3n - l4n;
                musum2 += sun * lun + sln * lln + s3n * l3n + s4n * l4n;
                rpmax = fmax(rpmax, fmax(fabs(kln + s3n - kb), fabs(-kln + s4n - kb)));
            }
            mu = block_reduce<0>(musum2, sh.red) / m4;
            rpmax = block_reduce<1>(rpmax, sh.red);
            __syncthreads();
            // dual residual r_d = E^T (kl - k_ref + l3 - l4) + f + lu - ll   (exact every iteration, O(N))
            apply_Et(slab, L, n, VV, ETV, t0, t1, t2, t3, t4, t5);
            rdmax = 0.0;
            if constexpr (PROX) {
                for (int i = threadIdx.x; i < n; i += IP_THREADS)
                    rdmax = fmax(rdmax, fabs(ETV[i] + prox_mu * AL[i] + F[i] + LU[i] - LL[i]));
            } else {
                for (int i = threadIdx.x; i < n; i += IP_THREADS) rdmax = fmax(rdmax, fabs(ETV[i] + F[i] + LU[i] - LL[i]));
            }
            rdmax = block_reduce<1>(rdmax, sh.red);
            if (mu <= prm.mu_rel * mu0 && rdmax <= rd_tol && rpmax <= 1e-8 * kb) { result = 0; ++it; break; }
            if (mu <= 1e-2 * prm.mu_rel * mu0) { result = (rdmax <= 1e3 * rd_tol && rpmax <= 1e-6 * kb) ? 0 : 2; ++it; break; }
        }
        write_instance<true>(aout, n, n_max, AL, b, result, it, status, iters_out);
    }
}

// ================================================================================================
// debug aid (tests/test_gpu_factor.py): factorise M = H + D of every instance with the fused forward substitution of
// V_RHS, solve into V_DX; then solve M x = V_T0 with the full sweeps into V_T1.  HB, V_DD, V_RHS, V_T0 are inputs.
// ================================================================================================
__global__ void __launch_bounds__(IP_THREADS, 8)
debug_factor_solve_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, double *__restrict__ ws, Layout L,
                          int32_t *__restrict__ status) {
    IpShared &sh = ip_init_shared();
    unsigned tick = 0;
    for (int b = blockIdx.x; b < B; b += gridDim.x) {
        const int n = n_pts ? n_pts[b] : n_max;
        double *slab = ws + (size_t)b * L.stride;
        if (threadIdx.x == 0) sh.flag = 0;
        __syncthreads();
        const bool ok = factor(sh, slab, L, n, slab + L.o_hb, vec(slab, L, V_RHS), tick);
        tick += factor_units(n);
        solve(sh, slab, L, n, vec(slab, L, V_RHS), vec(slab, L, V_DX), true);
        solve(sh, slab, L, n, vec(slab, L, V_T0), vec(slab, L, V_T1), false);
        // a second factorisation exercises the parity bookkeeping of the rings across calls
        const bool ok2 = factor(sh, slab, L, n, slab + L.o_hb, vec(slab, L, V_T0), tick);
        tick += factor_units(n);
        solve(sh, slab, L, n, vec(slab, L, V_T0), vec(slab, L, V_T2), true);
        if (threadIdx.x == 0) status[b] = (ok && ok2) ? 0 : 3;
        __syncthreads();
    }
}

// the width gradients of one instance (K2d, K2d') from v = (H + D + ...)^-1 g (X) and its box ratios DU, DL
__device__ __forceinline__ void width_grads(IpShared &sh, int n, int n_max, const double *__restrict__ rt, double wv,
                                            const double *__restrict__ DU, const double *__restrict__ DL,
                                            const double *__restrict__ X, double *__restrict__ gwr, double *__restrict__ gwl,
                                            double *__restrict__ gwv) {
    double gv = 0.0;
    for (int i = threadIdx.x; i < n_max; i += IP_THREADS) {
        double gr = 0.0, gl = 0.0;
        if (i < n) {
            const double v = X[i], gu = DU[i] * v, glb = DL[i] * v;
            const double2 ww = *reinterpret_cast<const double2 *>(rt + (size_t)i * 4 + 2);
            const double ub = ww.x - 0.5 * wv, lb = -(ww.y - 0.5 * wv);      // (the expressions of the setup)
            if (ub - lb < 2.0 * FIX_EPS) {
                gr = 0.5 * (gu + glb);
                gl = -gr;
            } else {
                gr = gu;
                gl = -glb;
                gv += 0.5 * (glb - gu);
            }
        }
        gwr[i] = gr;
        gwl[i] = gl;
    }
    gv = block_reduce<0>(gv, sh.red);
    if (threadIdx.x == 0) *gwv = gv;
}

// ================================================================================================
// K2d -- width sensitivities of the box-only QP (DESIGN.md section 3.10): implicit differentiation of its KKT conditions
// at the interior-point solution.  With the final ratios d_u = lu / su, d_l = ll / sl of the forward solve (`sens`,
// mincurv_sens_export_kernel) and an upstream gradient g of alpha:
//   (H + D) v = g,  D = d_u + d_l;   dL/dub = d_u v,  dL/dlb = d_l v
// and ub = w_right - w_veh / 2, lb = -w_left + w_veh / 2 (mincurv_setup_kernel P1).  A collapsed box (ub - lb < 2 FIX_EPS,
// replaced by mid -+ FIX_EPS) follows mid = (w_right - w_left) / 2: both widths get +-(dL/dub + dL/dlb) / 2, w_veh nothing.
// One factorisation and one solve per instance; the band of H is read from the owner's slab as in mincurv_pdip_kernel.
// Instances with grad_status != 0 get zeros; a non-positive pivot sets grad_status 3 (zeros too).
// ================================================================================================
__global__ void __launch_bounds__(IP_THREADS, 8)
mincurv_adjoint_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, const double *__restrict__ reftrack, double w_veh,
                       const double *__restrict__ w_veh_batch, double *__restrict__ ws, Layout L, const double *__restrict__ sens,
                       const double *__restrict__ grad_alpha, int32_t *__restrict__ grad_status,
                       double *__restrict__ grad_w_right, double *__restrict__ grad_w_left, double *__restrict__ grad_w_veh,
                       int *__restrict__ work_counter) {
    IpShared &sh = ip_init_shared();
    unsigned tick = 0;
    for (int b; (b = next_instance(sh, work_counter)) < B;) {
        const int n = n_pts ? n_pts[b] : n_max;
        double *gwr = grad_w_right + (size_t)b * n_max, *gwl = grad_w_left + (size_t)b * n_max;
        bool ok = grad_status[b] == 0;
        if (ok) {
            double *slab = ws + (size_t)b * L.stride;
            const double *HB = ws + (size_t)*band_owner(slab, L) * L.stride + L.o_hb;      // (shared centre lines: the owner's)
            const double *__restrict__ DU = sens + (size_t)b * 2 * n_max, *__restrict__ DL = DU + n_max;
            const double *__restrict__ GA = grad_alpha + (size_t)b * n_max;
            double *__restrict__ RHS = vec(slab, L, V_RHS), *__restrict__ DX = vec(slab, L, V_DX), *__restrict__ DD = vec(slab, L, V_DD);
            if (threadIdx.x == 0) sh.flag = 0;
            for (int i = threadIdx.x; i < L.np; i += IP_THREADS) {
                if (i < n) DD[i] = DU[i] + DL[i];
                RHS[i] = (i < n) ? GA[i] : 0.0;
            }
            ok = factor(sh, slab, L, n, HB, RHS, tick);
            tick += factor_units(n);
            if (ok) {
                solve(sh, slab, L, n, RHS, DX, true);
                width_grads(sh, n, n_max, reftrack + (size_t)b * n_max * 4, w_veh_batch ? w_veh_batch[b] : w_veh, DU, DL, DX,
                            gwr, gwl, grad_w_veh + b);
                continue;
            }
            if (threadIdx.x == 0) grad_status[b] = 3;
        }
        for (int i = threadIdx.x; i < n_max; i += IP_THREADS) { gwr[i] = 0.0; gwl[i] = 0.0; }
        if (threadIdx.x == 0) grad_w_veh[b] = 0.0;
    }
}

// ================================================================================================
// K2d' -- width sensitivities with the curvature rows (DESIGN.md section 3.10): the same iterate-based derivative at the
// final iterate of the curvature-row phase, whose KKT linearisation adds E^T W E, W = l3 / s3 + l4 / s4 (`sens_rows`,
// mincurv_sens_rows_export_kernel):
//   (H + D + E^T W E) v = g,   dL/dub = d_u v,  dL/dlb = d_l v
// W is split at 1, the weight of the objective's own rows in H = E^T I E.  The weak rows (W <= 1) stay in the band,
// K = E^T (I + W_weak) E + D (assembled into the instance's own slab, as the row phase does); the m strong rows S
// (W > 1: towards 1e12 at the row phase's end, where the band truncation is no longer SPD) are carried exactly by
// Woodbury:
//   Sigma = W_S^-1 + E_S K^-1 E_S^T (m x m, SPD, column j from one solve against E_S^T e_j; dense Cholesky in `schur`,
//           n_rows_cap^2 doubles per instance),   v = K^-1 g - K^-1 E_S^T Sigma^-1 E_S K^-1 g
// One factorisation, m + 2 solves, m + 1 applications each of E and E^T.  Instances with no row weight (solved by the
// box phase, or not solved) take the arithmetic of mincurv_adjoint_kernel.  pass 0 runs those, pass 1 the others: a
// row instance overwrites its own band of H, which followers of a shared centre line read in pass 0.  A non-positive
// pivot in K or in Sigma, or more strong rows than n_rows_cap, set grad_status 3 (zero gradients).
// ================================================================================================
__global__ void __launch_bounds__(IP_THREADS, 8)
mincurv_adjoint_rows_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, const double *__restrict__ reftrack,
                            double w_veh, const double *__restrict__ w_veh_batch, double *__restrict__ ws, Layout L,
                            const double *__restrict__ sens, const double *__restrict__ sens_rows,
                            const int32_t *__restrict__ n_rows, double *schur, int n_rows_cap, int pass,
                            const double *__restrict__ grad_alpha, int32_t *__restrict__ grad_status,
                            double *__restrict__ grad_w_right, double *__restrict__ grad_w_left, double *__restrict__ grad_w_veh,
                            int *__restrict__ work_counter) {
    IpShared &sh = ip_init_shared();
    unsigned tick = 0;
    for (int b; (b = next_instance(sh, work_counter)) < B;) {
        const int n = n_pts ? n_pts[b] : n_max;
        const double *__restrict__ WR = sens_rows + (size_t)b * n_max;
        double wmax = 0.0;
        for (int i = threadIdx.x; i < n_max; i += IP_THREADS) wmax = fmax(wmax, WR[i]);
        if ((block_reduce<1>(wmax, sh.red) > 0.0) != (pass == 1)) continue;      // (every row weight is > 0 where the row phase ran)
        double *gwr = grad_w_right + (size_t)b * n_max, *gwl = grad_w_left + (size_t)b * n_max;
        const double *rt = reftrack + (size_t)b * n_max * 4;
        const double wv = w_veh_batch ? w_veh_batch[b] : w_veh;
        const int m = n_rows[b];
        bool ok = grad_status[b] == 0 && m <= n_rows_cap;
        if (ok) {
            double *slab = ws + (size_t)b * L.stride;
            const double *__restrict__ DU = sens + (size_t)b * 2 * n_max, *__restrict__ DL = DU + n_max;
            const double *__restrict__ GA = grad_alpha + (size_t)b * n_max;
            double *RHS = vec(slab, L, V_RHS), *X = vec(slab, L, V_DX), *DD = vec(slab, L, V_DD), *WK = vec(slab, L, V_WK);
            if (threadIdx.x == 0) sh.flag = 0;
            if (pass == 0) {
                const double *HB = ws + (size_t)*band_owner(slab, L) * L.stride + L.o_hb;      // (shared centre lines: the owner's)
                for (int i = threadIdx.x; i < L.np; i += IP_THREADS) {
                    if (i < n) DD[i] = DU[i] + DL[i];
                    RHS[i] = (i < n) ? GA[i] : 0.0;
                }
                ok = factor(sh, slab, L, n, HB, RHS, tick);
                tick += factor_units(n);
                if (ok) solve(sh, slab, L, n, RHS, X, true);
            } else {
                double *R = vec(slab, L, V_T4K), *Y = vec(slab, L, V_RD), *Z = vec(slab, L, V_T3K), *EZ = vec(slab, L, V_EDX);
                double *U = vec(slab, L, V_VV);
                int *S = reinterpret_cast<int *>(vec(slab, L, V_ISU));      // the strong rows, ascending
                double *t0 = vec(slab, L, V_T0), *t1 = vec(slab, L, V_T1), *t2 = vec(slab, L, V_T2), *t3 = vec(slab, L, V_T3);
                double *t4 = vec(slab, L, V_T4), *t5 = vec(slab, L, V_T5);
                double *Sg = schur + (size_t)b * n_rows_cap * n_rows_cap;      // Sigma, row-major, lower triangle used
                for (int i = threadIdx.x; i < L.np; i += IP_THREADS) {
                    if (i < n) {
                        DD[i] = DU[i] + DL[i];
                        WK[i] = (WR[i] <= 1.0) ? WR[i] : 0.0;
                    }
                    RHS[i] = (i < n) ? GA[i] : 0.0;
                    R[i] = 0.0;
                }
                if (threadIdx.x < 32) {
                    const int lane = threadIdx.x;
                    int cnt = 0;
                    for (int base = 0; base < n; base += 32) {
                        const bool st = base + lane < n && WR[base + lane] > 1.0;
                        const unsigned bal = __ballot_sync(FULL, st);
                        if (st) S[cnt + __popc(bal & ((1u << lane) - 1u))] = base + lane;
                        cnt += __popc(bal);
                    }
                }
                __syncthreads();
                assemble_hband(slab, L, n, WK, sh.u.win);
                __syncthreads();
                ok = factor(sh, slab, L, n, slab + L.o_hb, RHS, tick);      // K, with the forward half of K^-1 g
                tick += factor_units(n);
                if (ok && m > 0) {
                    solve(sh, slab, L, n, RHS, X, true);
                    for (int j = 0; j < m; ++j) {      // column j of Sigma: E_S K^-1 E^T e_{S_j} + e_j / W_{S_j}
                        if (threadIdx.x == 0) R[S[j]] = 1.0;
                        __syncthreads();
                        apply_Et(slab, L, n, R, Y, t0, t1, t2, t3, t4, t5);
                        if (threadIdx.x == 0) R[S[j]] = 0.0;
                        solve(sh, slab, L, n, Y, Z, false);
                        apply_E(slab, L, n, Z, EZ, t0, t1, t2, t3, t4, t5);
                        for (int k = j + threadIdx.x; k < m; k += IP_THREADS)
                            Sg[(size_t)k * n_rows_cap + j] = EZ[S[k]] + ((k == j) ? 1.0 / WR[S[j]] : 0.0);
                    }
                    apply_E(slab, L, n, X, EZ, t0, t1, t2, t3, t4, t5);      // u = E_S K^-1 g
                    for (int k = threadIdx.x; k < m; k += IP_THREADS) U[k] = EZ[S[k]];
                    // Sigma = C C^T in place (right-looking, lower triangle)
                    for (int k = 0; k < m && ok; ++k) {
                        __syncthreads();
                        const double d = Sg[(size_t)k * n_rows_cap + k];
                        if (!(d > 0.0)) { ok = false; break; }
                        const double c = sqrt(d), ic = 1.0 / c;
                        __syncthreads();
                        if (threadIdx.x == 0) Sg[(size_t)k * n_rows_cap + k] = c;
                        for (int i = k + 1 + threadIdx.x; i < m; i += IP_THREADS) Sg[(size_t)i * n_rows_cap + k] *= ic;
                        __syncthreads();
                        const int r = m - k - 1;
                        for (int e = threadIdx.x; e < r * r; e += IP_THREADS) {
                            const int i = k + 1 + e / r, jj = k + 1 + e % r;
                            if (jj <= i) Sg[(size_t)i * n_rows_cap + jj] -= Sg[(size_t)i * n_rows_cap + k] * Sg[(size_t)jj * n_rows_cap + k];
                        }
                    }
                    if (ok) {
                        for (int k = 0; k < m; ++k) {          // C y = u
                            __syncthreads();
                            if (threadIdx.x == 0) U[k] /= Sg[(size_t)k * n_rows_cap + k];
                            __syncthreads();
                            const double yk = U[k];
                            for (int i = k + 1 + threadIdx.x; i < m; i += IP_THREADS) U[i] -= Sg[(size_t)i * n_rows_cap + k] * yk;
                        }
                        for (int k = m - 1; k >= 0; --k) {     // C^T z = y
                            __syncthreads();
                            if (threadIdx.x == 0) U[k] /= Sg[(size_t)k * n_rows_cap + k];
                            __syncthreads();
                            const double zk = U[k];
                            for (int i = threadIdx.x; i < k; i += IP_THREADS) U[i] -= Sg[(size_t)k * n_rows_cap + i] * zk;
                        }
                        __syncthreads();
                        for (int k = threadIdx.x; k < m; k += IP_THREADS) R[S[k]] = U[k];
                        __syncthreads();
                        apply_Et(slab, L, n, R, Y, t0, t1, t2, t3, t4, t5);      // v = K^-1 g - K^-1 E_S^T z
                        solve(sh, slab, L, n, Y, Z, false);
                        for (int i = threadIdx.x; i < n; i += IP_THREADS) X[i] -= Z[i];
                        __syncthreads();
                    }
                } else if (ok) {
                    solve(sh, slab, L, n, RHS, X, true);
                }
            }
            if (ok) {
                width_grads(sh, n, n_max, rt, wv, DU, DL, X, gwr, gwl, grad_w_veh + b);
                continue;
            }
        }
        if (threadIdx.x == 0 && grad_status[b] == 0) grad_status[b] = 3;
        for (int i = threadIdx.x; i < n_max; i += IP_THREADS) { gwr[i] = 0.0; gwl[i] = 0.0; }
        if (threadIdx.x == 0) grad_w_veh[b] = 0.0;
    }
}

// the curvature-row phase of mc_mincurv_kappa_batch (prox_mu 0) or of the projection QP of mc_mincurv_solve_batch_ex
// (Hessian H + prox_mu I, prox_mu > 0)
int mincurv_kappa_phase(int B, int n_max, const int32_t *n_pts, double kappa_bound, const double *kappa_bound_batch,
                        double prox_mu, double *alpha, int32_t *status, int32_t *iters, void *workspace,
                        size_t workspace_bytes, void *stream) {
    if (!alpha || !status) return bad("mc_mincurv_kappa_batch: NULL argument");
    int rc = mincurv_args("mc_mincurv_kappa_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    PdipParams prm;
    prm.max_iter = 40;
    prm.mu_rel = 1e-11;
    prm.rd_rel = 1e-8;
    prm.eta = 0.995;
    prm.dx_rel = 0.0;
    prm.lam0_rel = 1e-2;
    auto kernel = prox_mu > 0.0 ? mincurv_pdip_kappa_kernel<true> : mincurv_pdip_kappa_kernel<false>;
    const SolverGrid g = solver_grid(B, n_max, workspace, ctas_per_sm(kernel));
    if (launch_solver(kernel, g.grid, g.counter, (cudaStream_t)stream, B, n_max, n_pts, (double *)workspace,
                      make_layout(n_max), prm, kappa_bound, alpha, status, iters, g.counter, prox_mu,
                      kappa_bound_batch) != 0) {
        snprintf(g_err, sizeof(g_err), "mincurv_pdip_kappa_kernel: cudaFuncSetAttribute failed");
        return MC_ECUDA;
    }
    return check_cuda("mincurv_pdip_kappa_kernel");
}

}  // namespace mc

// the banded adjoint of mc_mincurv_adjoint_batch (K2d, or K2d' with sens_rows) after its argument checks
static int adjoint_banded(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                          const double *h, double w_veh, const double *w_veh_batch, double f_scale, const int32_t *centre_id,
                          const double *sens, int32_t *grad_status, const double *grad_alpha, double *grad_w_right,
                          double *grad_w_left, double *grad_w_veh, const double *sens_rows, const int32_t *n_rows,
                          double *schur, int n_rows_cap, const double *lin_alpha, void *workspace, size_t workspace_bytes,
                          void *stream) {
    // the band of H and the bounds are rebuilt in the slabs; the assembly's status words (the forward pass's, recorded in
    // grad_status) go to grad_w_right, which the adjoint kernel overwrites
    int rc = mc::mincurv_setup(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, centre_id, lin_alpha,
                               reinterpret_cast<int32_t *>(grad_w_right), workspace, workspace_bytes, stream);
    if (rc) return rc;
    if (sens_rows) {
        // pass 0: the instances without row weights (reading their owner's band); pass 1: the curvature-row instances
        const mc::SolverGrid g = mc::solver_grid(B, n_max, workspace, mc::ctas_per_sm(mc::mincurv_adjoint_rows_kernel));
        for (int pass = 0; pass < 2; ++pass) {
            if (mc::launch_solver(mc::mincurv_adjoint_rows_kernel, g.grid, g.counter, (cudaStream_t)stream, B, n_max, n_pts,
                                  reftrack, w_veh, w_veh_batch, (double *)workspace, mc::make_layout(n_max), sens, sens_rows,
                                  n_rows, schur, n_rows_cap, pass, grad_alpha, grad_status, grad_w_right, grad_w_left,
                                  grad_w_veh, g.counter) != 0) {
                snprintf(mc::g_err, sizeof(mc::g_err), "mincurv_adjoint_rows_kernel: cudaFuncSetAttribute failed");
                return MC_ECUDA;
            }
        }
        return check_cuda("mincurv_adjoint_rows_kernel");
    }
    const mc::SolverGrid g = mc::solver_grid(B, n_max, workspace, mc::ctas_per_sm(mc::mincurv_adjoint_kernel));
    if (mc::launch_solver(mc::mincurv_adjoint_kernel, g.grid, g.counter, (cudaStream_t)stream, B, n_max, n_pts, reftrack, w_veh,
                          w_veh_batch, (double *)workspace, mc::make_layout(n_max), sens, grad_alpha, grad_status, grad_w_right,
                          grad_w_left, grad_w_veh, g.counter) != 0) {
        snprintf(mc::g_err, sizeof(mc::g_err), "mincurv_adjoint_kernel: cudaFuncSetAttribute failed");
        return MC_ECUDA;
    }
    return check_cuda("mincurv_adjoint_kernel");
}

static constexpr int PDIP_SLICE_DEFAULT = 8;      // DESIGN.md section 3.3: the predictor of the remaining iterations is
                                                  // no better than chance after 4 iterations, within one iteration after 8

extern "C" {

int mc_mincurv_pdip_batch(int B, int n_max, const int32_t *n_pts, double *alpha, int32_t *status, int32_t *iters,
                          void *workspace, size_t workspace_bytes, void *stream) {
    if (!alpha || !status) return bad("mc_mincurv_pdip_batch: NULL argument");
    int rc = mc::mincurv_args("mc_mincurv_pdip_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    mc::PdipParams prm;
    prm.max_iter = 40;
    prm.mu_rel = 1e-10;
    prm.rd_rel = 1e-8;
    prm.eta = 0.995;
    prm.dx_rel = 1e-5;
    prm.lam0_rel = 1e-2;
    if (const char *e = getenv("MC_DEBUG_PDIP_LAM0")) { const double v = atof(e); if (v > 0.0) prm.lam0_rel = v; }   // start-point experiments only
    if (const char *e = getenv("MC_DEBUG_PDIP_ETA")) { const double v = atof(e); if (v > 0.5 && v < 1.0) prm.eta = v; }
    if (const char *e = getenv("MC_DEBUG_PDIP_DX_REL")) { const double v = atof(e); if (v >= 0.0) prm.dx_rel = v; }
    if (const char *e = getenv("MC_DEBUG_PDIP_MU_REL")) { const double v = atof(e); if (v > 0.0) prm.mu_rel = v; }   // tolerance experiments only
    int per_sm = mc::ctas_per_sm(mc::mincurv_pdip_kernel);
    if (const char *e = getenv("MC_DEBUG_PDIP_CTAS_PER_SM")) {      // occupancy experiments only (tools/prof_run.py)
        const int v = atoi(e);
        if (v > 0 && v < per_sm) per_sm = v;
    }
    // iterations before an instance is parked in the sliced schedule (DESIGN.md section 3.3); 0: every instance to the end
    int slice = PDIP_SLICE_DEFAULT;
    if (const char *e = getenv("MC_DEBUG_PDIP_SLICE")) { const int v = atoi(e); if (v >= 0) slice = v; }   // A/B runs and tests
    const mc::SolverGrid g = mc::solver_grid(B, n_max, workspace, per_sm);
    const mc::Layout L = mc::make_layout(n_max);
    double *ws = (double *)workspace;
    cudaStream_t s = (cudaStream_t)stream;
    // slice > 0 and more instances than CTAs: the sliced schedule (one launch, no grid-wide wait: the CTAs need not all be
    // resident); the schedule's ints sit behind the slabs
    if (B <= g.grid) slice = 0;
    cudaMemsetAsync(g.counter, 0, mc::SCHED_INTS * sizeof(int), s);
    if (slice > 0)      // the PARK_LIST entries of every slab
        cudaMemset2DAsync(ws + (size_t)mc::V_PARK * L.np + mc::PARK_LIST, L.stride * sizeof(double), 0,
                          mc::PARK_BUCKETS * sizeof(int), B, s);
    if (mc::launch_solver(mc::mincurv_pdip_kernel, g.grid, nullptr, s, B, n_max, n_pts, ws, L, prm, slice, alpha, status, iters,
                          g.counter) != 0) {
        snprintf(mc::g_err, sizeof(mc::g_err), "mincurv_pdip_kernel: cudaFuncSetAttribute failed");
        return MC_ECUDA;
    }
    return check_cuda("mincurv_pdip_kernel");
}

int mc_mincurv_kappa_batch(int B, int n_max, const int32_t *n_pts, double kappa_bound, double *alpha, int32_t *status,
                           int32_t *iters, const double *kappa_bound_batch, void *workspace, size_t workspace_bytes,
                           void *stream) {
    return mc::mincurv_kappa_phase(B, n_max, n_pts, kappa_bound, kappa_bound_batch, 0.0, alpha, status, iters, workspace,
                                   workspace_bytes, stream);
}

int mc_mincurv_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                             const double *h, double w_veh, const double *w_veh_batch, double f_scale, const int32_t *centre_id,
                             const double *sens, int32_t *grad_status, const double *grad_alpha, double *grad_w_right,
                             double *grad_w_left, double *grad_w_veh, const double *sens_rows, const int32_t *n_rows,
                             double *schur, int n_rows_cap, const double *lin_alpha, int dense_below, void *workspace,
                             size_t workspace_bytes, void *stream) {
    if (!sens || !grad_status || !grad_alpha || !grad_w_right || !grad_w_left || !grad_w_veh)
        return bad("mc_mincurv_adjoint_batch: NULL argument");
    if (sens_rows && (!n_rows || !schur)) return bad("mc_mincurv_adjoint_batch: sens_rows needs n_rows and schur");
    if (sens_rows && n_rows_cap < 0) return bad("mc_mincurv_adjoint_batch: n_rows_cap < 0");
    if (dense_below != 0) {
        if (dense_below < mc::N_MIN || dense_below > MC_DENSE_N_MAX + 1)
            return bad("mc_mincurv_adjoint_batch: dense_below must be 0 or in [%d, %d]", mc::N_MIN, MC_DENSE_N_MAX + 1);
        if (!sens_rows) return bad("mc_mincurv_adjoint_batch: dense_below needs sens_rows, n_rows and schur");
        if (lin_alpha) return bad("mc_mincurv_adjoint_batch: dense_below does not take lin_alpha");
        if (B <= 0 || n_max <= 0) return bad("mc_mincurv_adjoint_batch: B <= 0 or n_max <= 0");
        if (!reftrack || !normvec || !h) return bad("mc_mincurv_adjoint_batch: NULL argument");
    }
    // dense_below: the banded kernels run (if n_max >= N_MIN) with the dense adjoint's instances held out, then the dense one
    const bool banded = dense_below == 0 || n_max >= mc::N_MIN;
    if (banded) {
        int rc = 0;
        if (dense_below) {      // (the banded stage's own checks first: nothing is launched before every check passed)
            rc = mc::mincurv_args("mc_mincurv_adjoint_batch", B, n_max, workspace, workspace_bytes);
            if (!rc) rc = mc::mincurv_dense_hold(B, n_max, dense_below, n_pts, grad_status, stream);
            if (rc) return rc;
        }
        rc = adjoint_banded(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, centre_id, sens, grad_status,
                            grad_alpha, grad_w_right, grad_w_left, grad_w_veh, sens_rows, n_rows, schur, n_rows_cap, lin_alpha,
                            workspace, workspace_bytes, stream);
        if (rc || dense_below == 0) return rc;
    }
    return mc::mincurv_dense_adjoint(B, n_max, dense_below, banded, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale,
                                     centre_id, sens, grad_status, grad_alpha, grad_w_right, grad_w_left, grad_w_veh,
                                     sens_rows, n_rows, schur, n_rows_cap, stream);
}

/* debug aid (tests/test_gpu_factor.py): one factorisation + the two kinds of solve of the interior-point kernel on slabs
 * whose H band, V_DD, V_RHS and V_T0 the caller has filled in; results in V_DX, V_T1, V_T2 */
int mc_debug_factor_solve(int B, int n_max, const int32_t *n_pts, int32_t *status, void *workspace, size_t workspace_bytes,
                          void *stream) {
    if (!status) return bad("mc_debug_factor_solve: NULL argument");
    int rc = mc::mincurv_args("mc_debug_factor_solve", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    const mc::SolverGrid g = mc::solver_grid(B, n_max, workspace, mc::ctas_per_sm(mc::debug_factor_solve_kernel));
    if (mc::launch_solver(mc::debug_factor_solve_kernel, g.grid, nullptr, (cudaStream_t)stream, B, n_max, n_pts,
                          (double *)workspace, mc::make_layout(n_max), status) != 0)
        return bad("mc_debug_factor_solve: cudaFuncSetAttribute failed");
    return check_cuda("debug_factor_solve_kernel");
}

// debug aid: the cycle counters of CTA 0 of mincurv_pdip_kernel, slots as in enum ProfSlot; zeros unless built with
// -DMC_PROFILE
int mc_debug_read_profile(unsigned long long *host_out24, int reset) {
#ifdef MC_PROFILE
    if (cudaMemcpyFromSymbol(host_out24, mc::g_prof, sizeof(unsigned long long) * mc::PROF_SLOTS) != cudaSuccess) return MC_ECUDA;
    if (getenv("MC_PROFILE_SEGMENTS")) {       // tools/prof_run.py: sub-phase counters of one panel
        unsigned long long seg[32];
        if (cudaMemcpyFromSymbol(seg, mc::g_seg, sizeof(seg)) == cudaSuccess) {
            fprintf(stderr, "segments:");
            for (int i = 0; i < 32; ++i) fprintf(stderr, " %d:%llu", i, seg[i]);
            fprintf(stderr, "\n");
        }
    }
    if (reset) {
        unsigned long long z[32] = {0};
        if (cudaMemcpyToSymbol(mc::g_prof, z, sizeof(unsigned long long) * mc::PROF_SLOTS) != cudaSuccess) return MC_ECUDA;
        cudaMemcpyToSymbol(mc::g_seg, z, sizeof(z));
    }
    return MC_OK;
#else
    (void)reset;
    for (int i = 0; i < mc::PROF_SLOTS; ++i) host_out24[i] = 0ull;
    return MC_OK;
#endif
}

}  // extern "C"
