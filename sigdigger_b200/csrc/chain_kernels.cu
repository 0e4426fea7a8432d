// chain_kernels.cu -- per-channel inspector chains and Tasks/ primitives as serial recurrences, one
// GPU thread per (stream, channel) chain with the loop state carried in registers for the whole
// batch of channel samples (persistent across feeds through SdbChainState).
//
// COMPILED WITH -fmad=false: every expression below is a sequence of IEEE binary32 operations in
// source order, and the elementary functions are the fixed Cody-Waite + polynomial forms of
// SPEC.md section M, so soft symbols are bit-identical to the CPU oracle on identical input.
//
// Reference behaviour being replaced (all in suscan/sigutils, called from the reference at):
//   su_agc_feed            Tasks/AGCTask.cpp:70-73        su_costas_feed  Tasks/CostasRecoveryTask.cpp:58-61
//   su_pll_track           Tasks/PLLSyncTask.cpp:53-56    su_ncqo_read    Tasks/CarrierXlator.cpp:57-60
//   su_clock_detector_feed Tasks/WaveSampler.cpp:190-199  su_iir_filt_feed Tasks/WaveSampler.cpp:68-80
//   quadrature demod       Tasks/QuadDemodTask.cpp:44-60  Decider         Default/GenericInspector/InspectorUI.cpp:836-846
//   chain order            doc/SigDigger_User_Manual.pdf pp.50-52
#include "sdb_internal.h"
#include "../../include/sigdigger_b200.h"
#include <stdlib.h>
#include <string.h>

#include "sdb_chain_steps.h"
#include "sdb_cpx.h"

// ------------------------------------------------------------------ the chain kernel ------------
// One CTA = 32 chains (lane = chain) x 12 role warps.  A feed is cut into chunks of CH samples that move through
// eight pipeline steps, one CTA-wide barrier per iteration; a step that is feed-forward (every output depends only
// on inputs) is split over several warps by sample index, a step that is a true recurrence keeps one warp:
//
//   step  warps  role      work on its chunk                                                    hand-over
//   0     0      load      cp.async tile of the chunk (coalesced rows of the 32 chains)          tile[2]
//   1     1-2    pre       manual-offset LO, magnitude 10 log10 |y|^2 (8 samples per warp)       y[3], m[3]
//   2     0      track     AGC delay line swap, peak tracker, fast / slow levels (recurrence)     in place
//   3     3-4    post      gain 10^(level (slope - 1) / 20) x delayed sample; for ask + PLL also
//                          the phase detector's atan2 of the sample (feed-forward)               ringA[2], ang[2]
//   4     5      carrier   Costas | FSK discriminator | audio demod | ask: the PLL's phase / frequency
//                          recurrence only (recurrence)                                          ringB (circular), phs[2]
//   5     6-9    demod     ask: exp(-i phase), mix, component (|.| / I / Q), in place in ringB -- feed-forward
//                          once the phases are known (4 samples per warp)                        ringB
//   6     6-9    filter    matched filter: 4 outputs per warp straight off ringB (its history IS
//                          the filter line), two FFMAs per complex sample x tap; audio LPF (IIR, 1 warp) ringC[2]
//   7     10     clock     Gardner | sampler | resampler, CMA (recurrence)                       sym[2], cnt[2]
//   8     11     out       x0.75, decision (atan2 / modulus quantiser), symbol stores            global
//
// Feed-forward work runs beside the recurrences, not in series with them.  Loop state lives in registers for the
// whole feed, the per-chain lines in shared memory sized from the channel plan (SdbInspDyn).  Loops stay rolled:
// unrolled or per-class variants grow the code several-fold and starve the role warps on instruction fetch.
#define CH 16
enum { INSP_WARPS = 12 };              // role of each warp: see the dispatch at the end of k_inspectors
#define INSP_STEPS 8          // pipeline depth after the load: a chunk loaded in iteration c leaves in iteration c + 8

#ifdef SDB_STAGE_CYCLES
__device__ unsigned long long g_stage_cycles[8];
#define ROLE_T_DECL long long busy_ = 0
#define ROLE_T0 const long long t0_ = clock64()
#define ROLE_T1 busy_ += clock64() - t0_
__device__ unsigned long long g_role_cls[5][8];      // the same, by inspector class of the CTA
#define ROLE_T_END(slot) do { if (c.lane == 0) { atomicAdd(&g_stage_cycles[slot], (unsigned long long) busy_); \
  if (c.cls >= 0 && c.cls < 5) atomicAdd(&g_role_cls[c.cls][slot], (unsigned long long) busy_); } } while (0)
#else
#define ROLE_T_DECL
#define ROLE_T0
#define ROLE_T1
#define ROLE_T_END(slot)
#endif
// instrumented twin only: per inspector class c = 0..4: [c] sum of CTA lifetimes (cycles), [5 + c] CTAs,
// [10 + c] longest CTA (cycles), [15 + c] latest CTA end (ns, globaltimer), [20] earliest CTA start (ns)
#ifdef SDB_STAGE_CYCLES
__device__ unsigned long long g_cta_cycles[24];
#endif
cudaError_t sdb_stage_cta_cycles(unsigned long long out[64], int reset)
{
#ifdef SDB_STAGE_CYCLES
  cudaError_t e = cudaMemcpyFromSymbol(out, g_cta_cycles, sizeof(unsigned long long) * 24);
  if (e == cudaSuccess) e = cudaMemcpyFromSymbol(out + 24, g_role_cls, sizeof(unsigned long long) * 40);
  if (e == cudaSuccess && reset) {
    unsigned long long z[40] = { 0 };
    e = cudaMemcpyToSymbol(g_role_cls, z, sizeof(z));
    z[20] = ~0ull;
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_cta_cycles, z, sizeof(unsigned long long) * 24);
  }
  return e;
#else
  (void) reset;
  for (int i = 0; i < 64; ++i) out[i] = 0;
  return cudaSuccess;
#endif
}
cudaError_t sdb_stage_cycles(unsigned long long out[8], int reset)
{
#ifdef SDB_STAGE_CYCLES
  cudaError_t e = cudaMemcpyFromSymbol(out, g_stage_cycles, sizeof(unsigned long long) * 8);
  if (e == cudaSuccess && reset) {
    unsigned long long z[8] = { 0 };
    e = cudaMemcpyToSymbol(g_stage_cycles, z, sizeof(z));
  }
  return e;
#else
  (void) reset;
  for (int i = 0; i < 8; ++i) out[i] = 0;     // the counters are compiled out of the product build
  return cudaSuccess;
#endif
}
static __device__ __forceinline__ void cp_async8(void *smem_dst, const void *gsrc)
{
  const unsigned sa = (unsigned) __cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(sa), "l"(gsrc));
}
static __device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> static __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }
// CTA barrier reachable from the role functions (every role executes the same number of them)
static __device__ __forceinline__ void cta_sync()
{
  __syncwarp();                                  // bar.sync is warp-aligned: reconverge after the per-lane loops
  asm volatile("bar.sync 0;" ::: "memory");
}

struct ChainSmem {
  float2 tile[2][32][CH + 1];
  float2 y[3][CH][32];
  float  m[3][CH][32];
  float2 ringA[2][CH][32];
  float2 ringC[2][CH][32];
  float2 sym[2][CH][32];
  float  ang[2][CH][32];
  float  phs[2][CH][32];
  int    cnt[2][32];
};

// what every role needs to know about its lane's chain
struct ICtx {
  ChainSmem *sm;
  float2 (*rb)[32]; unsigned rb_mask;         // ringB: carrier output, circular, doubles as the matched-filter line
  float  (*taps)[32];                         // per-lane matched-filter taps [t][lane]
  float  (*agc)[32]; int agc_rows;
  float2 (*eqw)[32]; float2 (*eqx)[32];
  int lane, valid, cls, fresh;
  uint32_t n, nchunks;
  const SdbChainCfg *cp; SdbChainState *stp; float *bpool;
};

// SPEC E: constant-modulus equaliser on the symbol stream.  Sums and updates run in index order.
static __device__ __forceinline__ float2 cma_step(float2 (*w)[32], float2 (*x)[32], int lane, float mu,
                                                  int locked, float2 in)
{
#pragma unroll
  for (int i = SDB_EQ_LEN - 1; i > 0; --i) x[i][lane] = x[i - 1][lane];
  x[0][lane] = in;
  float yr = 0.0f, yi = 0.0f;
#pragma unroll
  for (int i = 0; i < SDB_EQ_LEN; ++i) {
    const float2 wi = w[i][lane], xi = x[i][lane];
    yr = yr + (wi.x * xi.x - wi.y * xi.y);
    yi = yi + (wi.x * xi.y + wi.y * xi.x);
  }
  if (!locked) {
    const float y2 = yr * yr + yi * yi;
    const float er = yr * (y2 - 1.0f), ei = yi * (y2 - 1.0f);
#pragma unroll
    for (int i = 0; i < SDB_EQ_LEN; ++i) {
      const float2 xi = x[i][lane];
      float2 wi = w[i][lane];
      const float gr = xi.x * er + xi.y * ei;
      const float gi = xi.x * ei - xi.y * er;
      wi.x = wi.x - mu * gr;
      wi.y = wi.y - mu * gi;
      w[i][lane] = wi;
    }
  }
  return make_float2(yr, yi);
}

// ---- steps 0 + 2: tile loader and AGC tracker (warp 0)
static __device__ void role_track(const ICtx &c, const float2 *chan_row)
{
  ChainSmem &sm = *c.sm;
  const int lane = c.lane;
  const SdbChainCfg *cp = c.cp; SdbChainState *stp = c.stp;
  const bool have_agc = c.valid && cp->have_agc && c.cls != SDB_INSP_RAW;
  float far_ = 0, faf = 0, sar = 0, saf = 0; unsigned hang_max = 0, dl_size = 1, mh_size = 1;
  AgcS as; as.fast = as.slow = as.peak = -160.0f; as.hang_n = as.dl_ptr = as.mh_ptr = 0;
  float *dl = nullptr, *mh = nullptr; bool in_smem = false;
  // the delay line is a pure delay (feed-forward): with the lines in shared memory and at least a chunk long, the
  // two pre warps swap their own samples through it (distinct slots within a chunk) and this warp keeps only the
  // level tracker, the recurrence (role_pre)
  bool dl_in_pre = false; unsigned dl_ptr0 = 0;
  if (have_agc) {
    far_ = cp->far_; faf = cp->faf; sar = cp->sar; saf = cp->saf;
    hang_max = cp->hang_max; dl_size = cp->dl_size; mh_size = cp->mh_size;
    as.fast = stp->fast_level; as.slow = stp->slow_level; as.peak = stp->peak;
    as.hang_n = stp->hang_n; as.dl_ptr = stp->dl_ptr; as.mh_ptr = stp->mh_ptr;
    in_smem = 2 * dl_size + mh_size <= (unsigned) c.agc_rows;
    dl_in_pre = in_smem && dl_size >= CH;
    dl_ptr0 = as.dl_ptr;
    float *gdl = c.bpool + (size_t) cp->st_dl_off * 32, *gmh = c.bpool + (size_t) cp->st_mh_off * 32;
    if (in_smem) {
      dl = &c.agc[0][lane]; mh = &c.agc[2 * dl_size][lane];
      for (unsigned i = 0; i < 2 * dl_size; ++i) dl[i * 32] = c.fresh ? 0.0f : gdl[i * 32];
      for (unsigned i = 0; i < mh_size; ++i) mh[i * 32] = c.fresh ? -160.0f : gmh[i * 32];
    } else {
      dl = gdl; mh = gmh;
      if (c.fresh) {
        for (unsigned i = 0; i < 2 * dl_size; ++i) dl[i * 32] = 0.0f;
        for (unsigned i = 0; i < mh_size; ++i) mh[i * 32] = -160.0f;
      }
    }
  }
  // coalesced, asynchronous tile load: row r of the tile = CH consecutive samples of the CTA's chain r; a warp
  // instruction copies two rows (16 lanes x 8 bytes = 128 contiguous bytes each)
  const unsigned long long rowp = (unsigned long long) chan_row;
  const uint32_t n = c.n;
  const int col = lane & (CH - 1), rsel = lane / CH;
  auto issue_tile = [&](uint32_t ch) {
    const uint32_t b0 = ch * CH;
#pragma unroll 8
    for (int j = 0; j < 32 / (32 / CH); ++j) {
      const int r = j * (32 / CH) + rsel;
      const unsigned long long pr = __shfl_sync(0xffffffffu, rowp, r);
      const uint32_t nr = __shfl_sync(0xffffffffu, n, r);
      if (b0 + col < nr) cp_async8(&sm.tile[ch & 1][r][col], (const float2 *) pr + b0 + col);
    }
    cp_async_commit();
  };
  const uint32_t total = c.nchunks + INSP_STEPS;
  ROLE_T_DECL;
  for (uint32_t it = 0; it <= total; ++it) {
    ROLE_T0;
    if (it < c.nchunks) issue_tile(it);
    if (have_agc && it >= 2 && it - 2 < c.nchunks) {
      const uint32_t ck = it - 2, base = ck * CH;
      const int b3 = (int) (ck % 3u);
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      auto run = [&](float *dl_, float *mh_) {
        if (dl_in_pre) {
          for (int i = 0; i < cnt; ++i)
            sm.m[b3][i][lane] = agc_level_sel<32>(far_, faf, sar, saf, hang_max, mh_size, as, mh_, sm.m[b3][i][lane]);
          return;
        }
        for (int i = 0; i < cnt; ++i) {
          // delay line: the sample that entered dl_size samples ago leaves, this one takes its slot
          const float2 y = sm.y[b3][i][lane];
          const unsigned dp = as.dl_ptr;
          as.dl_ptr = dp + 1 >= dl_size ? 0 : dp + 1;
          const float2 xd = make_float2(dl_[(2 * dp) * 32], dl_[(2 * dp + 1) * 32]);
          dl_[(2 * dp) * 32] = y.x; dl_[(2 * dp + 1) * 32] = y.y;
          sm.y[b3][i][lane] = xd;
          // magnitude history, running peak, fast / slow levels (SPEC A), select form
          sm.m[b3][i][lane] = agc_level_sel<32>(far_, faf, sar, saf, hang_max, mh_size, as, mh_, sm.m[b3][i][lane]);
        }
      };
      // lines in shared memory (the usual case): pointers the compiler can see are shared, so LDS / STS and not
      // generic loads and stores (the merged `in_smem ? shared : global` pointer made every access generic)
      if (in_smem) run(&c.agc[0][lane], &c.agc[2 * dl_size][lane]);
      else         run(dl, mh);
    }
    cp_async_wait<0>();
    ROLE_T1;
    cta_sync();
  }
  ROLE_T_END(0);
#ifdef SDB_STAGE_CYCLES
  if (lane == 0) {
    atomicAdd(&g_stage_cycles[4], (unsigned long long) c.nchunks * CH);
    if (c.cls >= 0 && c.cls < 5) atomicAdd(&g_role_cls[c.cls][4], (unsigned long long) c.nchunks * CH);
  }
#endif
  if (have_agc) {
    if (dl_in_pre) as.dl_ptr = (dl_ptr0 + c.n % dl_size) % dl_size;     // where the pre warps left it
    stp->fast_level = as.fast; stp->slow_level = as.slow; stp->peak = as.peak;
    stp->hang_n = as.hang_n; stp->dl_ptr = as.dl_ptr; stp->mh_ptr = as.mh_ptr;
    if (in_smem) {
      float *gdl = c.bpool + (size_t) cp->st_dl_off * 32, *gmh = c.bpool + (size_t) cp->st_mh_off * 32;
      for (unsigned i = 0; i < 2 * dl_size; ++i) gdl[i * 32] = dl[i * 32];
      for (unsigned i = 0; i < mh_size; ++i) gmh[i * 32] = mh[i * 32];
    }
  }
}

// ---- step 1: manual-offset LO + magnitude in dB (warps 1-2, half a chunk each)
static __device__ void role_pre(const ICtx &c, int part)
{
  ChainSmem &sm = *c.sm;
  const int lane = c.lane;
  const bool have_agc = c.valid && c.cp->have_agc && c.cls != SDB_INSP_RAW;
  const bool have_lo = c.valid && c.cls != SDB_INSP_AUDIO && c.cp->have_lo;
  float lo_phi = have_lo ? c.stp->lo_phi : 0.0f;
  const float lo_omega = have_lo ? c.cp->lo_omega : 0.0f;
  const uint32_t n = c.n, total = c.nchunks + INSP_STEPS;
  const int i0 = part * (CH / 2), i1 = i0 + CH / 2;
  // AGC delay line (SPEC A: the sample that entered dl_size samples ago leaves, the new one takes its slot): a pure
  // delay, so each pre warp swaps its own half of the chunk -- sample i of the chunk uses slot (start + i) mod dl_size,
  // distinct within a chunk when dl_size >= CH.  Same condition as in role_track, which then skips the line.
  unsigned dl_size = 1, dl_base = 0;
  bool dl_here = false;
  if (have_agc) {
    dl_size = c.cp->dl_size;
    dl_here = 2 * dl_size + c.cp->mh_size <= (unsigned) c.agc_rows && dl_size >= CH;
    dl_base = c.stp->dl_ptr;                      // (read before role_track rewrites it at the end of the kernel)
  }
  float *dl = &c.agc[0][lane];
  auto through_delay = [&](int i, float2 y) -> float2 {
    unsigned sl = dl_base + (unsigned) i;
    if (sl >= dl_size) sl -= dl_size;
    const float2 xd = make_float2(dl[(2 * sl) * 32], dl[(2 * sl + 1) * 32]);
    dl[(2 * sl) * 32] = y.x; dl[(2 * sl + 1) * 32] = y.y;
    return xd;
  };
  __syncwarp();
  ROLE_T_DECL;
  for (uint32_t it = 0; it <= total; ++it) {
    ROLE_T0;
    if (it >= 1 && it - 1 < c.nchunks) {
      const uint32_t ck = it - 1, base = ck * CH;
      const int b3 = (int) (ck % 3u);
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      float2 (*tl)[CH + 1] = sm.tile[ck & 1];
      if (have_lo) {
        // both pre warps run the (cheap) phase recurrence over the whole chunk and evaluate exp(i phi) only for
        // their own samples: phi is the same sequence of binary32 additions as in the serial statement
        for (int i = 0; i < cnt; ++i) {
          if (i >= i0 && i < i1) {
            float s, co;
            d_sincosf(lo_phi, &s, &co);
            float2 y = tl[lane][i];
            y = make_float2(y.x * co + y.y * s, y.y * co - y.x * s);
            sm.y[b3][i][lane] = dl_here ? through_delay(i, y) : y;
            if (have_agc) sm.m[b3][i][lane] = 10.0f * d_log10f(y.x * y.x + y.y * y.y + 1e-16f);
          }
          lo_phi = wrap_once(lo_phi + lo_omega);
        }
      } else {
#pragma unroll 4
        for (int i = i0; i < i1; ++i) {
          if (i < cnt) {
            const float2 y = tl[lane][i];
            sm.y[b3][i][lane] = dl_here ? through_delay(i, y) : y;
            if (have_agc) sm.m[b3][i][lane] = 10.0f * d_log10f(y.x * y.x + y.y * y.y + 1e-16f);
          }
        }
      }
      if (dl_here) { dl_base += (unsigned) cnt; if (dl_base >= dl_size) dl_base -= dl_size; }
    }
    ROLE_T1;
    cta_sync();
  }
  if (part == 0) ROLE_T_END(5);
  if (have_lo && part == 0) c.stp->lo_phi = lo_phi;
}

// ---- step 3: gain (warps 3-4, half a chunk each)
static __device__ void role_post(const ICtx &c, int part)
{
  ChainSmem &sm = *c.sm;
  const int lane = c.lane, cls = c.cls;
  const bool have_agc = c.valid && c.cp->have_agc && cls != SDB_INSP_RAW;
  const float knee = c.valid ? c.cp->knee : 0.0f, slope_m1 = c.valid ? c.cp->gain_slope - 1.0f : 0.0f;
  const float fixed_gain = c.valid ? c.cp->fixed_gain : 1.0f;
  const float gain2 = (c.valid && cls != SDB_INSP_AUDIO) ? c.cp->gain2 : 1.0f;
  const uint32_t n = c.n, total = c.nchunks + INSP_STEPS;
  const int i0 = part * (CH / 2), i1 = i0 + CH / 2;
  // ask + PLL: the phase detector's atan2 depends on the sample alone, not on the loop: evaluated here, beside the
  // recurrence instead of inside it (same function on the same argument: bit-identical to pll_step)
  const bool want_ang = c.valid && cls == SDB_INSP_ASK && c.cp->have_pll;
  // the usual CTA -- every chain a symbol inspector behind an AGC, all or none of them wanting the angle -- on a full
  // chunk: the statements below without their per-sample guards (the general loop spends 8 branches per sample on
  // them), 1 = gain only, 2 = gain + angle
  int fast = 0;
  if (__all_sync(0xffffffffu, !c.valid || (have_agc && cls != SDB_INSP_AUDIO)))
    fast = __all_sync(0xffffffffu, !c.valid || want_ang) ? 2 : (__all_sync(0xffffffffu, !want_ang) ? 1 : 0);
  ROLE_T_DECL;
  for (uint32_t it = 0; it <= total; ++it) {
    ROLE_T0;
    const bool active = it >= 3 && it - 3 < c.nchunks;
    const bool full_chunk = active && fast && __all_sync(0xffffffffu, !c.valid || ((it - 3) * CH + CH <= n));
    if (full_chunk) {
      const uint32_t ck = it - 3;
      const int b3 = (int) (ck % 3u);
      float2 (*out)[32] = sm.ringA[ck & 1];
      float (*ang)[32] = sm.ang[ck & 1];
#pragma unroll 4
      for (int i = i0; i < i1; ++i) {
        float2 y = sm.y[b3][i][lane];
        const float lvl = sm.m[b3][i][lane];
        const float gx = d_db_to_mag(lvl * slope_m1);
        float g = lvl < knee ? fixed_gain : gx;
        g = g * 0.7f;
        y.x = y.x * g; y.y = y.y * g;
        y.x = 2.0f * y.x; y.y = 2.0f * y.y;
        out[i][lane] = y;
        if (fast == 2) ang[i][lane] = d_atan2f(y.y, y.x);
      }
    } else if (active) {
      const uint32_t ck = it - 3, base = ck * CH;
      const int b3 = (int) (ck % 3u);
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      float2 (*out)[32] = sm.ringA[ck & 1];
      float (*ang)[32] = sm.ang[ck & 1];
#pragma unroll 4
      for (int i = i0; i < i1; ++i) {
        if (i < cnt) {
          float2 y = sm.y[b3][i][lane];
          if (have_agc) {
            const float lvl = sm.m[b3][i][lane];
            float g = lvl < knee ? fixed_gain : d_db_to_mag(lvl * slope_m1);
            g = g * 0.7f;
            y.x = y.x * g; y.y = y.y * g;
            if (cls != SDB_INSP_AUDIO) { y.x = 2.0f * y.x; y.y = 2.0f * y.y; }
          } else if (cls != SDB_INSP_RAW && cls != SDB_INSP_AUDIO) {
            y.x = gain2 * y.x; y.y = gain2 * y.y;
          }
          out[i][lane] = y;
          if (want_ang) ang[i][lane] = d_atan2f(y.y, y.x);
        }
      }
    }
    ROLE_T1;
    cta_sync();
  }
  if (part == 0) ROLE_T_END(6);
}

// ---- step 4: carrier stage (warp 5)
static __device__ void role_carrier(const ICtx &c)
{
  ChainSmem &sm = *c.sm;
  const int lane = c.lane, cls = c.cls;
  const SdbChainCfg *cp = c.cp; SdbChainState *stp = c.stp;
  CostasK ck; CostasS cs; float p_phi = 0, p_omega = 0, pll_a = 0, pll_b = 0, prev_re = 0, prev_im = 0;
  float rot_re = 1, rot_im = 0, dc = 0, sq_level = 0, dc_alpha = 0, sq_alpha = 0, sq_thr = 0, lo_phi = 0, lo_omega = 0;
  int have_costas = 0, have_pll = 0, quad = 0, ask_ch = 0, ademod = 0, asquelch = 0;
  ck.kind = 0; ck.af_n = 1; ck.a = ck.b = 0;
  cs.phi = cs.omega = cs.lock = cs.yre = cs.yim = 0;
#pragma unroll
  for (int i = 0; i < SDB_MAX_IIR; ++i) { ck.af_b[i] = ck.af_a[i] = 0; cs.xr[i] = cs.xi[i] = cs.yr[i] = cs.yi[i] = 0; }
  if (c.valid) {
    have_costas = cp->have_costas; have_pll = cp->have_pll;
    ck.kind = cp->costas_kind; ck.af_n = cp->af_n; ck.a = cp->c_a; ck.b = cp->c_b;
#pragma unroll
    for (int i = 0; i < SDB_MAX_IIR; ++i) {
      ck.af_b[i] = cp->af_b[i]; ck.af_a[i] = cp->af_a[i];
      cs.xr[i] = stp->afx_re[i]; cs.xi[i] = stp->afx_im[i]; cs.yr[i] = stp->afy_re[i]; cs.yi[i] = stp->afy_im[i];
    }
    cs.phi = stp->c_phi; cs.omega = stp->c_omega; cs.lock = stp->c_lock; cs.yre = stp->c_yre; cs.yim = stp->c_yim;
    p_phi = stp->p_phi; p_omega = stp->p_omega; pll_a = cp->pll_alpha; pll_b = cp->pll_beta;
    prev_re = stp->prev_re; prev_im = stp->prev_im;
    rot_re = cp->fsk_rot_re; rot_im = cp->fsk_rot_im; quad = cp->fsk_quad_demod; ask_ch = cp->ask_channel;
    ademod = cp->audio_demod; asquelch = cp->audio_squelch; dc = stp->dc; sq_level = stp->sq_level;
    dc_alpha = cp->dc_alpha; sq_alpha = cp->sq_alpha; sq_thr = cp->sq_thr;
    if (cls == SDB_INSP_AUDIO) { lo_phi = stp->lo_phi; lo_omega = cp->lo_omega; }
  }
  // Costas: when every chain of the warp runs the same loop kind and arm-filter length (the usual case: a CTA holds
  // one inspector class), the sample loop is the compile-time variant -- no per-lane branches between the dependent
  // operations of the recurrence, which is the slowest role of the psk CTAs (988 cycles per sample with them)
  int psk_sel = 0;
  {
    const unsigned vm = __ballot_sync(0xffffffffu, c.valid != 0);
    const int src = vm ? __ffs(vm) - 1 : 0;
    const int kind0 = __shfl_sync(0xffffffffu, ck.kind, src), afn0 = __shfl_sync(0xffffffffu, ck.af_n, src);
    const int hc0 = __shfl_sync(0xffffffffu, have_costas, src);
    const bool same = __all_sync(0xffffffffu, !c.valid || (ck.kind == kind0 && ck.af_n == afn0 && have_costas == hc0));
    if (cls == SDB_INSP_PSK && same && hc0 && kind0 >= 1 && kind0 <= 3 && (afn0 == 1 || afn0 == 3))
      psk_sel = kind0 * 4 + afn0;
  }
  // the same for the other classes: one compact loop per class when the warp is uniform (1: ask + PLL, 2: fsk).  The
  // general loop below branches over every class per sample; its body is several hundred instructions long and the
  // jumps between its far-apart blocks showed up as instruction-fetch stalls on the warp that sets the CTA's pace.
  int uni_sel = 0;
  if (__all_sync(0xffffffffu, !c.valid || (cls == SDB_INSP_ASK && have_pll))) uni_sel = 1;
  const int quad_u = __shfl_sync(0xffffffffu, quad, __ffs(__ballot_sync(0xffffffffu, c.valid != 0) | 0x80000000u) - 1);
  if (!uni_sel && __all_sync(0xffffffffu, !c.valid || (cls == SDB_INSP_FSK && quad == quad_u))) uni_sel = 2;
  const uint32_t n = c.n, total = c.nchunks + INSP_STEPS;
  ROLE_T_DECL;
  for (uint32_t it = 0; it <= total; ++it) {
    ROLE_T0;
    if (psk_sel && it >= 4 && it - 4 < c.nchunks) {
      const uint32_t ckk = it - 4, base = ckk * CH;
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      float2 (*in)[32] = sm.ringA[ckk & 1];
#define PSK_LOOP(K_, A_) for (int i = 0; i < cnt; ++i) \
        c.rb[(base + i) & c.rb_mask][lane] = costas_step_t<K_, A_>(ck, cs, in[i][lane]); break
      switch (psk_sel) {
        case 1 * 4 + 1: PSK_LOOP(1, 1);
        case 1 * 4 + 3: PSK_LOOP(1, 3);
        case 2 * 4 + 1: PSK_LOOP(2, 1);
        case 2 * 4 + 3: PSK_LOOP(2, 3);
        case 3 * 4 + 1: PSK_LOOP(3, 1);
        default:        PSK_LOOP(3, 3);
      }
#undef PSK_LOOP
    } else if (uni_sel == 1 && it >= 4 && it - 4 < c.nchunks) {
      // ask + PLL, every chain of the warp: the (phi, omega) recurrence alone (see the general loop below)
      const uint32_t ckk = it - 4, base = ckk * CH;
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      float2 (*in)[32] = sm.ringA[ckk & 1];
      float (*ang)[32] = sm.ang[ckk & 1], (*phs)[32] = sm.phs[ckk & 1];
      for (int i = 0; i < cnt; ++i) {
        phs[i][lane] = p_phi;
        p_phi = wrap_once(p_phi + p_omega);
        float err = ang[i][lane] - p_phi;
        err = err > PI_F ? err - TWOPI_F : (err < -PI_F ? err + TWOPI_F : err);
        p_omega = p_omega + pll_a * err;
        p_phi = wrap_once(p_phi + pll_b * err);
        c.rb[(base + i) & c.rb_mask][lane] = in[i][lane];
      }
    } else if (uni_sel == 2 && it >= 4 && it - 4 < c.nchunks) {
      // fsk, every chain of the warp: the discriminator alone
      const uint32_t ckk = it - 4, base = ckk * CH;
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      float2 (*in)[32] = sm.ringA[ckk & 1];
      for (int i = 0; i < cnt; ++i) {
        float2 y = in[i][lane];
        const float dr = y.x * prev_re + y.y * prev_im;
        const float di = y.y * prev_re - y.x * prev_im;
        prev_re = y.x; prev_im = y.y;
        if (quad_u) { y.x = d_atan2f(di, dr) * 0.318309886183790671538f; y.y = 0.0f; }     // warp-uniform
        else { y.x = dr * rot_re - di * rot_im; y.y = dr * rot_im + di * rot_re; }
        c.rb[(base + i) & c.rb_mask][lane] = y;
      }
    } else if (it >= 4 && it - 4 < c.nchunks) {
      const uint32_t ckk = it - 4, base = ckk * CH;
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      float2 (*in)[32] = sm.ringA[ckk & 1];
      for (int i = 0; i < cnt; ++i) {
        float2 y = in[i][lane];
        if (cls == SDB_INSP_PSK) {
          if (have_costas) y = costas_step(ck, cs, y);
        } else if (cls == SDB_INSP_FSK) {
          float dr = y.x * prev_re + y.y * prev_im;
          float di = y.y * prev_re - y.x * prev_im;
          prev_re = y.x; prev_im = y.y;
          if (quad) { y.x = d_atan2f(di, dr) * 0.318309886183790671538f; y.y = 0.0f; }
          else { y.x = dr * rot_re - di * rot_im; y.y = dr * rot_im + di * rot_re; }
        } else if (cls == SDB_INSP_ASK) {
          // Only (phi, omega) is a recurrence: phi <- wrap(phi + omega); err = wrap(ang - phi); omega += alpha err;
          // phi <- wrap(phi + beta err) -- pll_step statement by statement.  The oscillator read exp(i phi), the mix
          // and the component selection need this sample's phase only and run in the demod step (role_filter).
          if (have_pll) {
            sm.phs[ckk & 1][i][lane] = p_phi;
            p_phi = wrap_once(p_phi + p_omega);
            float err = sm.ang[ckk & 1][i][lane] - p_phi;
            if (err > PI_F) err = err - TWOPI_F;
            else if (err < -PI_F) err = err + TWOPI_F;
            p_omega = p_omega + pll_a * err;
            p_phi = wrap_once(p_phi + pll_b * err);
          }
        } else if (cls == SDB_INSP_AUDIO) {
          float v = 0.0f;
          float p = y.x * y.x + y.y * y.y;
          sq_level = sq_level + sq_alpha * (p - sq_level);
          if (ademod == SDB_AUDIO_AM) {
            v = d_cabsf(y.x, y.y);
            dc = dc + dc_alpha * (v - dc);
            v = v - dc;
          } else if (ademod == SDB_AUDIO_FM) {
            float dr = y.x * prev_re + y.y * prev_im;
            float di = y.y * prev_re - y.x * prev_im;
            v = d_atan2f(di, dr) * 0.318309886183790671538f;
            prev_re = y.x; prev_im = y.y;
          } else if (ademod == SDB_AUDIO_USB || ademod == SDB_AUDIO_LSB) {
            float2 ph = ncqo_read(lo_phi, lo_omega);
            v = y.x * ph.x - y.y * ph.y;
          }
          if (asquelch && !(sq_level > sq_thr)) v = 0.0f;
          y = make_float2(v, 0.0f);
        }
        c.rb[(base + i) & c.rb_mask][lane] = y;
      }
    }
    ROLE_T1;
    cta_sync();
  }
  ROLE_T_END(1);
  if (c.valid) {
#pragma unroll
    for (int i = 0; i < SDB_MAX_IIR; ++i) {
      stp->afx_re[i] = cs.xr[i]; stp->afx_im[i] = cs.xi[i]; stp->afy_re[i] = cs.yr[i]; stp->afy_im[i] = cs.yi[i];
    }
    stp->c_phi = cs.phi; stp->c_omega = cs.omega; stp->c_lock = cs.lock; stp->c_yre = cs.yre; stp->c_yim = cs.yim;
    stp->p_phi = p_phi; stp->p_omega = p_omega; stp->prev_re = prev_re; stp->prev_im = prev_im;
    stp->dc = dc; stp->sq_level = sq_level;
    if (cls == SDB_INSP_AUDIO) stp->lo_phi = lo_phi;
  }
}

// ---- step 5: matched filter / audio low-pass (warps 6-9, a quarter of a chunk each)
// The carrier ring IS the filter line: output p needs x[p - t], t < mf_n, which are the mf_n most recent ring
// entries (the last mf_n - 1 samples of the previous feed are put back in front of position 0 at kernel start).
// One thread produces 4 consecutive outputs of its chain from a sliding register window: per tap one ring load,
// one tap load and four complex-by-real FMAs (complex sample x real tap, SPEC I.1: ascending taps, fused terms).
static __device__ void role_filter(const ICtx &c, int part, const float *taps_pool)
{
  ChainSmem &sm = *c.sm;
  const int lane = c.lane;
  const SdbChainCfg *cp = c.cp; SdbChainState *stp = c.stp;
  const int have_mf = c.valid ? cp->have_mf : 0, mf_n = c.valid ? cp->mf_n : 0;
  const int alpf_n = (c.valid && c.cls == SDB_INSP_AUDIO) ? cp->alpf_n : 0;
  const bool mf_ring = have_mf && (unsigned) (mf_n - 1 + 3 * CH) <= c.rb_mask + 1u;
  const bool mf_global = have_mf && !mf_ring;
  const uint32_t n = c.n, total = c.nchunks + INSP_STEPS;
  float al_b[SDB_MAX_IIR], al_a[SDB_MAX_IIR], al_x[SDB_MAX_IIR], al_xi[SDB_MAX_IIR], al_y[SDB_MAX_IIR], al_yi[SDB_MAX_IIR];
  unsigned mf_ptr = 0; float *mfl = nullptr; const float *gtaps = nullptr;
  if (part == 0) {
#pragma unroll
    for (int i = 0; i < SDB_MAX_IIR; ++i) {
      al_b[i] = c.valid ? cp->alpf_b[i] : 0.0f; al_a[i] = c.valid ? cp->alpf_a[i] : 0.0f;
      al_x[i] = c.valid ? stp->al_x[i] : 0.0f; al_y[i] = c.valid ? stp->al_y[i] : 0.0f;
      al_xi[i] = 0.0f; al_yi[i] = 0.0f;
    }
    if (mf_ring) {
      const float *tp = taps_pool + cp->mf_off;
      const float *gmf = c.bpool + (size_t) cp->st_mf_off * 32;
      for (int t = 0; t < mf_n; ++t) c.taps[t][lane] = __ldg(tp + t);
      for (int k2 = 1; k2 < mf_n; ++k2)       // x[-k2]: the k2-th newest sample of the previous feed
        c.rb[(0u - (unsigned) k2) & c.rb_mask][lane] =
            c.fresh ? make_float2(0.f, 0.f) : make_float2(gmf[(2 * (k2 - 1)) * 32], gmf[(2 * (k2 - 1) + 1) * 32]);
    } else if (mf_global) {
      // filters too long for the ring keep a circular line in the global pool and run serially on one warp
      gtaps = taps_pool + cp->mf_off; mf_ptr = stp->mf_ptr;
      mfl = c.bpool + (size_t) cp->st_mf_off * 32;
      if (c.fresh) for (int i = 0; i < 2 * mf_n; ++i) mfl[i * 32] = 0.0f;
    }
  }
  const bool ask = c.valid && c.cls == SDB_INSP_ASK;
  const bool ask_pll = ask && cp->have_pll;
  const int ask_ch = ask ? cp->ask_channel : 0;
  ROLE_T_DECL;
  for (uint32_t it = 0; it <= total; ++it) {
    ROLE_T0;
    // ---- step 5, ask only: finish the carrier stage of chunk it - 5 in place (4 samples per warp)
    if (ask && it >= 5 && it - 5 < c.nchunks) {
      const uint32_t ck = it - 5, base = ck * CH;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int i = part * 4 + j;
        const uint32_t p = base + (uint32_t) i;
        if (p < n) {
          float2 y = c.rb[p & c.rb_mask][lane];
          if (ask_pll) {
            float sn, cs;
            d_sincosf(sm.phs[ck & 1][i][lane], &sn, &cs);            // the NCQO read of pll_step
            y = make_float2(y.x * cs + y.y * sn, y.y * cs - y.x * sn);
          }
          if (ask_ch == 0)      { y.x = d_cabsf(y.x, y.y); y.y = 0.0f; }
          else if (ask_ch == 1) { y.y = 0.0f; }
          else                  { y.x = y.y; y.y = 0.0f; }
          c.rb[p & c.rb_mask][lane] = y;
        }
      }
    }
    // ---- step 6: filter chunk it - 6
    if (it >= 6 && it - 6 < c.nchunks) {
      const uint32_t ck = it - 6, base = ck * CH;
      float2 (*out)[32] = sm.ringC[ck & 1];
      if (mf_ring) {
        const uint32_t p0 = base + (uint32_t) part * 4u;
        if (p0 < n) {
          float2 a0 = make_float2(0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
          float2 w0 = c.rb[(p0 + 0) & c.rb_mask][lane], w1 = c.rb[(p0 + 1) & c.rb_mask][lane];
          float2 w2 = c.rb[(p0 + 2) & c.rb_mask][lane], w3 = c.rb[(p0 + 3) & c.rb_mask][lane];
          // tap t needs ring entry (p0 - 1 - t) mod ring: two linear runs (before / after the ring's wrap), so the
          // loads are [pointer + immediate] instead of a mask and a shift per load (the address arithmetic was
          // 20 of the 45 instructions of a 4-tap trip, on the one role that can fill a scheduler's issue slots)
          const unsigned q = (p0 - 1u) & c.rb_mask;
          const float2 *xp = &c.rb[q][lane];               // rows are 32 float2 apart
          const float *tp = &c.taps[0][lane];
          int t = 0;
#define MF_TAP(o_) { const float b = tp[(o_) * 32]; const float2 bb = make_float2(b, b); const float2 nx = xp[-(o_) * 32]; \
            a0 = sdb_fma2(bb, w0, a0); a1 = sdb_fma2(bb, w1, a1); a2 = sdb_fma2(bb, w2, a2); a3 = sdb_fma2(bb, w3, a3); \
            w3 = w2; w2 = w1; w1 = w0; w0 = nx; }
#define MF_RUN(end_) { _Pragma("unroll 1") for (; t + 4 <= (end_); t += 4) { MF_TAP(0) MF_TAP(1) MF_TAP(2) MF_TAP(3) xp -= 4 * 32; tp += 4 * 32; } \
            _Pragma("unroll 1") for (; t < (end_); ++t) { MF_TAP(0) xp -= 32; tp += 32; } }
          const int t_wrap = mf_n < (int) q + 1 ? mf_n : (int) q + 1;
          MF_RUN(t_wrap)
          xp += (size_t) (c.rb_mask + 1u) * 32;
          MF_RUN(mf_n)
#undef MF_RUN
#undef MF_TAP
          const int j0 = part * 4;
          out[j0][lane] = a0;
          if (p0 + 1 < n) out[j0 + 1][lane] = a1;
          if (p0 + 2 < n) out[j0 + 2][lane] = a2;
          if (p0 + 3 < n) out[j0 + 3][lane] = a3;
        }
      } else if (mf_global || alpf_n > 0) {
        if (part == 0) {
          const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
          for (int i = 0; i < cnt; ++i) {
            float2 y = c.rb[(base + i) & c.rb_mask][lane];
            if (mf_global) {
              float accr = 0.0f, acci = 0.0f;
              mfl[(2 * mf_ptr) * 32] = y.x; mfl[(2 * mf_ptr + 1) * 32] = y.y;
              unsigned p = mf_ptr;
              for (int t = 0; t < mf_n; ++t) {
                const float b = __ldg(gtaps + t);
                accr = __fmaf_rn(b, mfl[(2 * p) * 32], accr);
                acci = __fmaf_rn(b, mfl[(2 * p + 1) * 32], acci);
                p = p == 0 ? mf_n - 1 : p - 1;
              }
              mf_ptr = mf_ptr + 1 == (unsigned) mf_n ? 0 : mf_ptr + 1;
              y = make_float2(accr, acci);
            } else {
              y = iir_any(alpf_n, al_b, al_a, al_x, al_xi, al_y, al_yi, y);
            }
            out[i][lane] = y;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t p = base + (uint32_t) (part * 4 + j);
          if (p < n) out[part * 4 + j][lane] = c.rb[p & c.rb_mask][lane];
        }
      }
    }
    ROLE_T1;
    cta_sync();
  }
  if (part == 0) ROLE_T_END(2);
  if (part == 0 && c.valid) {
#pragma unroll
    for (int i = 0; i < SDB_MAX_IIR; ++i) { stp->al_x[i] = al_x[i]; stp->al_y[i] = al_y[i]; }
    if (mf_ring) {
      float *gmf = c.bpool + (size_t) cp->st_mf_off * 32;
      for (int k2 = 1; k2 < mf_n; ++k2) {
        const float2 v = c.rb[(n - (unsigned) k2) & c.rb_mask][lane];
        gmf[(2 * (k2 - 1)) * 32] = v.x; gmf[(2 * (k2 - 1) + 1) * 32] = v.y;
      }
    } else if (mf_global) {
      stp->mf_ptr = mf_ptr;
    }
  }
}

// ---- step 6: clock recovery / sampler / resampler, CMA (warp 10).  Emits the chunk's symbols (before the x0.75
// and the decision) into sym[] and their number into cnt[]; the out role finishes them.
static __device__ void role_clock(const ICtx &c)
{
  ChainSmem &sm = *c.sm;
  const int lane = c.lane, cls = c.cls;
  const SdbChainCfg *cp = c.cp; SdbChainState *stp = c.stp;
  ClockS ks; float clk_gain = 0, clk_alpha = 0, clk_beta = 0, smp_period = 0, smp_phase0 = 0, s_phase = 0, s_pr = 0, s_pi = 0;
  int clock_type = 1, clock_running = 1;
  float avol = 1, rs_prev = 0; double rs_step = 0, rs_phase = 0;
  int eq_type = 0, eq_locked = 0; float eq_mu = 0;
  ks.phi = ks.bnor = ks.x0r = ks.x0i = ks.x1r = ks.x1i = ks.x2r = ks.x2i = ks.pr = ks.pi = 0; ks.half = 0;
  if (c.valid) {
    ks.phi = stp->k_phi; ks.bnor = stp->k_bnor; ks.x0r = stp->k_x0r; ks.x0i = stp->k_x0i; ks.x1r = stp->k_x1r;
    ks.x1i = stp->k_x1i; ks.x2r = stp->k_x2r; ks.x2i = stp->k_x2i; ks.pr = stp->k_pr; ks.pi = stp->k_pi;
    ks.half = stp->k_half;
    clk_gain = cp->clk_gain; clk_alpha = cp->clk_alpha; clk_beta = cp->clk_beta;
    smp_period = cp->smp_period; smp_phase0 = cp->smp_phase0; s_phase = stp->s_phase; s_pr = stp->s_pr; s_pi = stp->s_pi;
    clock_type = cp->clock_type; clock_running = cp->clock_running;
    avol = cp->audio_volume; rs_prev = stp->rs_prev; rs_step = cp->rs_step; rs_phase = stp->rs_phase;
    eq_type = cp->eq_type; eq_locked = cp->eq_locked; eq_mu = cp->eq_mu;
    if (eq_type == 1) {
      for (int i = 0; i < SDB_EQ_LEN; ++i) {
        c.eqw[i][lane] = make_float2(stp->eq_wr[i], stp->eq_wi[i]);
        c.eqx[i][lane] = make_float2(stp->eq_xr[i], stp->eq_xi[i]);
      }
    }
  }
  // every chain of the warp a symbol inspector on the Gardner loop without equaliser (the usual CTA): the sample
  // loop is the select form of clock_step alone, with none of the other classes' state live in it
  const bool gardner_only = __all_sync(0xffffffffu, !c.valid || (cls != SDB_INSP_RAW && cls != SDB_INSP_AUDIO &&
                                                               clock_type == 1 && eq_type == 0));
  const uint32_t n = c.n, total = c.nchunks + INSP_STEPS;
  ROLE_T_DECL;
  for (uint32_t it = 0; it <= total; ++it) {
    ROLE_T0;
    if (gardner_only && it >= 7 && it - 7 < c.nchunks) {
      const uint32_t ck = it - 7, base = ck * CH;
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      float2 (*in)[32] = sm.ringC[ck & 1];
      float2 (*sy)[32] = sm.sym[ck & 1];
      int k = 0;
      for (int i = 0; i < cnt; ++i) {
        float2 o;
        const bool produced = clock_step_sel(clk_gain, clk_alpha, clk_beta, ks, in[i][lane], o);
        if (produced && clock_running) sy[k++][lane] = o;
      }
      sm.cnt[ck & 1][lane] = k;
    } else if (it >= 7 && it - 7 < c.nchunks) {
      const uint32_t ck = it - 7, base = ck * CH;
      const int cnt = base >= n ? 0 : (n - base < CH ? (int) (n - base) : CH);
      float2 (*in)[32] = sm.ringC[ck & 1];
      float2 (*sy)[32] = sm.sym[ck & 1];
      int k = 0;
      for (int i = 0; i < cnt; ++i) {
        float2 y = in[i][lane], o;
        if (cls == SDB_INSP_RAW) {
          sy[k++][lane] = y;
        } else if (cls == SDB_INSP_AUDIO) {
          rs_phase += rs_step;
          if (rs_phase >= 1.0) {
            rs_phase -= 1.0;
            float al = (float) (rs_phase / rs_step);
            if (al > 1.0f) al = 1.0f;
            sy[k++][lane] = make_float2(avol * ((1.0f - al) * y.x + al * rs_prev), 0.0f);
          }
          rs_prev = y.x;
        } else {
          bool produced;
          if (clock_type == 1) produced = clock_step(clk_gain, clk_alpha, clk_beta, ks, y, o);
          else                 produced = sampler_step(smp_period, smp_phase0, s_phase, s_pr, s_pi, y, o);
          if (produced && eq_type == 1) o = cma_step(c.eqw, c.eqx, lane, eq_mu, eq_locked, o);
          if (produced && clock_running) sy[k++][lane] = o;
        }
      }
      sm.cnt[ck & 1][lane] = k;
    }
    ROLE_T1;
    cta_sync();
  }
  ROLE_T_END(3);
  if (c.valid) {
    stp->k_phi = ks.phi; stp->k_bnor = ks.bnor; stp->k_x0r = ks.x0r; stp->k_x0i = ks.x0i; stp->k_x1r = ks.x1r;
    stp->k_x1i = ks.x1i; stp->k_x2r = ks.x2r; stp->k_x2i = ks.x2i; stp->k_pr = ks.pr; stp->k_pi = ks.pi;
    stp->k_half = ks.half; stp->s_phase = s_phase; stp->s_pr = s_pr; stp->s_pi = s_pi;
    stp->rs_prev = rs_prev; stp->rs_phase = rs_phase;
    if (eq_type == 1) {
      for (int i = 0; i < SDB_EQ_LEN; ++i) {
        stp->eq_wr[i] = c.eqw[i][lane].x; stp->eq_wi[i] = c.eqw[i][lane].y;
        stp->eq_xr[i] = c.eqx[i][lane].x; stp->eq_xi[i] = c.eqx[i][lane].y;
      }
    }
  }
}

// ---- step 7: -2.5 dB, decision, symbol stores (warp 11; feed-forward, off the clock recurrence)
static __device__ void role_out(const ICtx &c, float2 *__restrict__ so, unsigned char *__restrict__ ho,
                                uint32_t *__restrict__ sym_count, size_t sym_cap)
{
  ChainSmem &sm = *c.sm;
  const int lane = c.lane, cls = c.cls;
  int dec_mode = 0, dec_int = 1; float dec_min = 0, dec_h = 1;
  if (c.valid) { dec_mode = c.cp->dec_mode; dec_int = c.cp->dec_intervals; dec_min = c.cp->dec_min; dec_h = c.cp->dec_h; }
  const bool decided = cls != SDB_INSP_RAW && cls != SDB_INSP_AUDIO;
  uint32_t nout = 0;
  const uint32_t total = c.nchunks + INSP_STEPS;
  for (uint32_t it = 0; it <= total; ++it) {
    if (it >= 8 && it - 8 < c.nchunks) {
      const uint32_t ck = it - 8;
      const int k = c.valid ? sm.cnt[ck & 1][lane] : 0;
      float2 (*sy)[32] = sm.sym[ck & 1];
      for (int j = 0; j < k; ++j) {
        if (nout < sym_cap) {
          float2 o = sy[j][lane];
          unsigned char h = 0;
          if (decided) {
            o.x = 0.75f * o.x; o.y = 0.75f * o.y;
            h = decide(dec_mode, dec_min, dec_h, dec_int, o);
          }
          so[nout] = o; ho[nout] = h;
          ++nout;
        }
      }
    }
    cta_sync();
  }
  if (c.valid) *sym_count = nout;
}

__global__ void __launch_bounds__(INSP_WARPS * 32, 2) k_inspectors(const SdbChainCfg *__restrict__ cfgs, int n_channels,
                                                     int n_streams, const int *__restrict__ chain_map,
                                                     SdbChainState *__restrict__ states,
                                                     float *__restrict__ pool, size_t pool_stride,
                                                     const float *__restrict__ taps_pool,
                                                     const SdbChannelDev *__restrict__ chans,
                                                     const float2 *__restrict__ chan_in,
                                                     size_t chan_stream_stride, uint32_t n_hops,
                                                     float2 *__restrict__ soft, unsigned char *__restrict__ hard,
                                                     uint32_t *__restrict__ sym_counts, size_t sym_cap, int fresh,
                                                     const SdbInspDyn dyn)
{
  extern __shared__ __align__(16) unsigned char smem_raw[];
  ICtx c;
  c.sm = reinterpret_cast<ChainSmem *>(smem_raw);
  unsigned char *dp = smem_raw + sizeof(ChainSmem);
  c.rb = reinterpret_cast<float2 (*)[32]>(dp); dp += (size_t) dyn.rb_slots * 32 * sizeof(float2);
  c.rb_mask = (unsigned) dyn.rb_slots - 1u;
  c.taps = reinterpret_cast<float (*)[32]>(dp); dp += (size_t) dyn.mf_rows * 32 * sizeof(float);
  c.agc = reinterpret_cast<float (*)[32]>(dp); dp += (size_t) dyn.agc_rows * 32 * sizeof(float);
  c.agc_rows = dyn.agc_rows;
  c.eqw = reinterpret_cast<float2 (*)[32]>(dp); c.eqx = c.eqw + SDB_EQ_LEN;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int chains = n_channels * n_streams;
  const int slot = blockIdx.x * 32 + lane;
  // chain_map: CTA slot -> channel-major chain index k * S + s, or -1 (padding so that a CTA holds one class)
  const int g = chain_map ? chain_map[slot] : (slot < chains ? slot : -1);
  const bool valid = g >= 0;
  const int k = valid ? g / n_streams : 0, s = valid ? g - k * n_streams : 0;
  const int chain = s * n_channels + k;                // index into states / outputs (stream-major)
  c.lane = lane; c.valid = valid ? 1 : 0; c.fresh = fresh;
  c.cp = cfgs + k; c.stp = states + chain;
  c.cls = valid ? c.cp->cls : -1;
  c.n = valid ? n_hops * (uint32_t) chans[k].halfsz : 0;
  c.bpool = pool + (size_t) blockIdx.x * 32 * pool_stride + lane;     // per-CTA pool, interleaved [slot][lane]
  __shared__ uint32_t s_nmax;
  if (threadIdx.x == 0) s_nmax = 0;
  __syncthreads();
  if (warp == 0) atomicMax(&s_nmax, c.n);
  __syncthreads();
  c.nchunks = (s_nmax + CH - 1) / CH;
#ifdef SDB_STAGE_CYCLES
  const long long cta_t0 = clock64();
  unsigned long long cta_ns0;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(cta_ns0));
#endif

  // Role of each warp.  Warps go to the SM's four schedulers by warp index modulo 4, and the matched filter is the one
  // role that can issue every cycle (independent FFMAs): three of its four warps share scheduler 1 among themselves,
  // so that the recurrence warps (track, carrier -- the roles that set the CTA's pace) never compete with one for
  // an issue slot:  scheduler 0: track, pre 0, out;  1: filter 0-2;  2: carrier, pre 1, post 0;  3: clock, post 1, filter 3
  // (one call site per role with the part as a run-time value: a call per warp index would inline four copies of the
  // filter role and two of pre / post, and the kernel, at 290 KB of code, ran three times slower)
  const unsigned role = ((dyn.role_lut ? dyn.role_lut : 0x343641315230ull) >> (4 * warp)) & 15u;   // nibble w: role of warp w
  const unsigned part = ((dyn.role_lut ? dyn.part_lut : 0x302011100000ull) >> (4 * warp)) & 15u;   //           its part
  if (role == 0) {
    role_track(c, valid ? chan_in + (size_t) s * chan_stream_stride + chans[k].out_off : nullptr);
  } else if (role == 1) {
    role_pre(c, (int) part);
  } else if (role == 2) {
    role_carrier(c);
  } else if (role == 3) {
    role_filter(c, (int) part, taps_pool);
  } else if (role == 4) {
    role_post(c, (int) part);
  } else if (role == 5) {
    role_clock(c);
  } else {
    role_out(c, soft + (size_t) chain * sym_cap, hard + (size_t) chain * sym_cap, sym_counts + chain, sym_cap);
  }
#ifdef SDB_STAGE_CYCLES
  __syncthreads();
  if (threadIdx.x == 0 && c.cls >= 0 && c.cls < 5) {
    const unsigned long long el = (unsigned long long) (clock64() - cta_t0);
    unsigned long long ns1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns1));
    atomicAdd(&g_cta_cycles[c.cls], el);
    atomicAdd(&g_cta_cycles[5 + c.cls], 1ull);
    atomicMax(&g_cta_cycles[10 + c.cls], el);
    atomicMax(&g_cta_cycles[15 + c.cls], ns1);
    atomicMin(&g_cta_cycles[20], cta_ns0);
  }
#endif
}

size_t sdb_inspector_smem_bytes(const SdbInspDyn &dyn)
{
  return sizeof(ChainSmem) + (size_t) dyn.rb_slots * 32 * sizeof(float2) + (size_t) dyn.mf_rows * 32 * sizeof(float) +
         (size_t) dyn.agc_rows * 32 * sizeof(float) + (dyn.use_eq ? 2 * (size_t) SDB_EQ_LEN * 32 * sizeof(float2) : 0);
}

cudaError_t sdb_launch_inspectors_n(const SdbLaunchCtx &c, const SdbChainCfg *cfg_dev, int n_channels,
                                    int n_streams, const int *chain_map, int n_ctas, SdbChainState *state,
                                    float *pool, size_t pool_stride,
                                    const float *taps_pool, const SdbChannelDev *chans_dev,
                                    const float2 *chan_in, size_t chan_stream_stride, uint32_t n_hops,
                                    float2 *soft, uint8_t *hard, uint32_t *sym_counts, size_t sym_cap, int fresh,
                                    const SdbInspDyn &dyn)
{
  const int chains = n_channels * n_streams;
  if (chains == 0) return cudaSuccess;
  static std::atomic<unsigned long long> attr_done{ 0 };   // one bit per device: function attributes are per context
  if (sdb_first_on_device(attr_done))
    cudaFuncSetAttribute(k_inspectors, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);   // + static < 227 KB
  const size_t smem = sdb_inspector_smem_bytes(dyn);
  if (!chain_map) n_ctas = (chains + 31) / 32;
  // SDB_INSP_PLACEMENT=linear: roles in warp order (track, pre x2, post x2, carrier, filter x4, clock, out), the
  // placement of the first builds -- kept for A/B measurements
  static const bool linear = getenv("SDB_INSP_PLACEMENT") && !strcmp(getenv("SDB_INSP_PLACEMENT"), "linear");
  SdbInspDyn d2 = dyn;
  if (linear) { d2.role_lut = 0x653333244110ull; d2.part_lut = 0x3210010100ull; }
  k_inspectors<<<n_ctas, INSP_WARPS * 32, smem, c.stream>>>(
      cfg_dev, n_channels, n_streams, chain_map, state, pool, pool_stride, taps_pool, chans_dev, chan_in,
      chan_stream_stride, n_hops, soft, hard, sym_counts, sym_cap, fresh, d2);
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}

// ------------------------------------------------------------------ Tasks/ primitives -----------
// One thread per buffer of the batch; same recurrences, state in registers.
__global__ void k_task_xlate(const float2 *__restrict__ src, float2 *__restrict__ dst, size_t n, size_t batch,
                             float omega, float phi0)
{
  size_t b = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (b >= batch) return;
  float phi = phi0;
  const float2 *x = src + b * n;
  float2 *y = dst + b * n;
  for (size_t i = 0; i < n; ++i) {
    float2 ph = ncqo_read(phi, omega);
    float2 v = x[i];
    y[i] = make_float2(v.x * ph.x - v.y * ph.y, v.x * ph.y + v.y * ph.x);
  }
}

// quadrature demod has no loop-carried state beyond x[p-1]: fully parallel over samples
__global__ void k_task_quad(const float2 *__restrict__ src, float2 *__restrict__ dst, size_t n, size_t batch)
{
  size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (i >= n * batch) return;
  size_t p = i % n;
  if (p == 0) { dst[i] = make_float2(0.0f, 0.0f); return; }
  float2 x = src[i], pv = src[i - 1];
  float dr = x.x * pv.x + x.y * pv.y;
  float di = x.y * pv.x - x.x * pv.y;
  dst[i] = make_float2(0.0f, 0.318309886183790671538f * d_atan2f(di, dr));
}

// mode 0 Costas, 1 PLL, 2 AGC.  pool: per-buffer AGC arrays, interleaved by 32 buffers ([slot][lane]).
__global__ void k_task_chain(const float2 *__restrict__ src, float2 *__restrict__ dst, size_t n, size_t batch,
                             const SdbChainCfg *__restrict__ cp, int mode, float *pool, size_t pool_stride)
{
  size_t b = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (b >= batch) return;
  const float2 *x = src + b * n;
  float2 *y = dst + b * n;
  if (mode == 0) {
    CostasK ck; CostasS cs;
    ck.kind = cp->costas_kind; ck.af_n = cp->af_n; ck.a = cp->c_a; ck.b = cp->c_b;
#pragma unroll
    for (int i = 0; i < SDB_MAX_IIR; ++i) {
      ck.af_b[i] = cp->af_b[i]; ck.af_a[i] = cp->af_a[i];
      cs.xr[i] = cs.xi[i] = cs.yr[i] = cs.yi[i] = 0.0f;
    }
    cs.phi = cs.omega = cs.lock = cs.yre = cs.yim = 0.0f;
    for (size_t i = 0; i < n; ++i) y[i] = costas_step(ck, cs, x[i]);
  } else if (mode == 1) {
    float phi = 0.0f, omega = 0.0f;
    const float a = cp->pll_alpha, be = cp->pll_beta;
    for (size_t i = 0; i < n; ++i) y[i] = pll_step(a, be, phi, omega, x[i]);
  } else {
    AgcK ak; AgcS as;
    ak.knee = cp->knee; ak.slope_m1 = cp->gain_slope - 1.0f; ak.fixed_gain = cp->fixed_gain;
    ak.far_ = cp->far_; ak.faf = cp->faf; ak.sar = cp->sar; ak.saf = cp->saf;
    ak.hang_max = cp->hang_max; ak.dl_size = cp->dl_size; ak.mh_size = cp->mh_size;
    as.fast = as.slow = as.peak = -160.0f; as.hang_n = as.dl_ptr = as.mh_ptr = 0;
    float *bp = pool + (b / 32) * 32 * pool_stride + (b % 32);
    float *dl = bp + (size_t) cp->st_dl_off * 32, *mh = bp + (size_t) cp->st_mh_off * 32;
    for (unsigned i = 0; i < 2 * ak.dl_size; ++i) dl[i * 32] = 0.0f;
    for (unsigned i = 0; i < ak.mh_size; ++i) mh[i * 32] = -160.0f;
    for (size_t i = 0; i < n; ++i) y[i] = agc_step(ak, as, dl, mh, x[i]);
  }
}

// One buffer, loop state handed in and out (the bulk twins of su_costas_feed / su_pll_track: a Tasks/ work()
// block continues where the previous one stopped).  mode 0: st = CostasK ++ CostasS, 1: st = {alpha, beta, phi, omega}
__global__ void k_task_chain_state(const float2 *__restrict__ x, float2 *__restrict__ y, size_t n, int mode,
                                   float *__restrict__ st)
{
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  if (mode == 0) {
    CostasK ck = *reinterpret_cast<const CostasK *>(st);
    CostasS cs = *reinterpret_cast<const CostasS *>(reinterpret_cast<const unsigned char *>(st) + sizeof(CostasK));
    for (size_t i = 0; i < n; ++i) y[i] = costas_step(ck, cs, x[i]);
    *reinterpret_cast<CostasS *>(reinterpret_cast<unsigned char *>(st) + sizeof(CostasK)) = cs;
  } else {
    const float a = st[0], be = st[1];
    float phi = st[2], omega = st[3];
    for (size_t i = 0; i < n; ++i) y[i] = pll_step(a, be, phi, omega, x[i]);
    st[2] = phi; st[3] = omega;
  }
}
cudaError_t sdb_launch_task_chain_state(cudaStream_t s, const float2 *src, float2 *dst, size_t n, int mode, float *st)
{
  k_task_chain_state<<<1, 32, 0, s>>>(src, dst, n, mode, st);
  return cudaGetLastError();
}
size_t sdb_costas_k_bytes(void) { return sizeof(CostasK); }
size_t sdb_costas_s_bytes(void) { return sizeof(CostasS); }

cudaError_t sdb_launch_task_xlate(cudaStream_t s, const float2 *src, float2 *dst, size_t n, size_t batch,
                                  float omega, float phi0)
{
  k_task_xlate<<<(unsigned) ((batch + 31) / 32), 32, 0, s>>>(src, dst, n, batch, omega, phi0);
  return cudaGetLastError();
}
cudaError_t sdb_launch_task_quad(cudaStream_t s, const float2 *src, float2 *dst, size_t n, size_t batch)
{
  size_t tot = n * batch;
  k_task_quad<<<(unsigned) ((tot + 255) / 256), 256, 0, s>>>(src, dst, n, batch);
  return cudaGetLastError();
}
cudaError_t sdb_launch_task_chain(cudaStream_t s, const float2 *src, float2 *dst, size_t n, size_t batch,
                                  const SdbChainCfg *cfg_dev, int mode, float *pool, size_t pool_stride)
{
  k_task_chain<<<(unsigned) ((batch + 31) / 32), 32, 0, s>>>(src, dst, n, batch, cfg_dev, mode, pool, pool_stride);
  return cudaGetLastError();
}
