// fac_kernels.cu -- the inspector's FAC tab (oracle/SPEC_FC.md; Default/GenericInspector/FACTab.cpp): the averaged,
// peak-marked autocorrelation of each FAC chain's soft symbols, in blocks of L = 2^9 .. 2^19 symbols.
//
// Symbol counts exist only on the device, so one feed runs a fixed sequence of launches whatever it completes:
//   k_fac_plan     counts + each chain's fill p -> the blocks this feed completes, as per-chain prefix sums of four
//                  kinds of work unit (F.2 blocks, F.3 4096-point units, 1024-lag statistics tiles, averaging units);
//   k_fac_small    L <= 4096: one CTA per block, F.2 forward, P = |X|^2, F.2 inverse, v = |A| (FC.1);
//   k_fac_cols/rows L >= 8192: the F.3 column and row passes, twice (FC.1: |A| = |F_L(P)|), through a per-block
//                  scratch, each pass in units of 4096 points;
//   k_fac_tilemax  per tile of the lag window: max, min and first arg-max of v;
//   k_fac_prefix   per chain: the running maximum entering each tile, in one pass over the feed's tiles;
//   k_fac_tilepow  per tile: the excluded records and the FC.2 tree sum;
//   k_fac_fixup    per chain, serially over its blocks: localMax, pos, power, count, max, min and the status (FC.4);
//   k_fac_average  per chain and 1024 lags: fac += alpha (v / max - fac), block by block (FC.3);
//   k_fac_tail     per chain: the symbols past the last completed block become the carried block.
// Every unit kernel is a persistent grid that walks the units of the feed and exits when there are none, so a feed
// that completes no block costs a few near-empty launches.  Built with -fmad=false: the only fused operations are the
// explicit __fmaf_rn of SPEC F.1, and every FC.2 / FC.3 operation is a round-to-nearest intrinsic.
#include "sdb_internal.h"
#include "sdb_math.h"
#include "sdb_fft_block.h"
#include <math_constants.h>

#define FAC_THREADS 256
#define FAC_TILE 1024

// the last chain c with off[c] <= u (off nondecreasing, off[0] = 0 <= u < off[C])
static __device__ __forceinline__ int fac_find(const uint32_t *__restrict__ off, int C, uint32_t u)
{
  int lo = 0, hi = C;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= u) lo = mid; else hi = mid;
  }
  return lo;
}

// element i of block j of a chain: the carried block below the fill p, the feed's symbols after it
static __device__ __forceinline__ float2 fac_in(const float2 *__restrict__ blk, const float2 *__restrict__ soft,
                                                uint32_t j, uint32_t L, uint32_t p, uint32_t i)
{
  const long long g = (long long) j * L + i - p;
  return g < 0 ? blk[i] : soft[g];
}

// exclusive sum over the CTA of FAC_THREADS threads; `total` gets the sum of all
static __device__ __forceinline__ uint32_t fac_exscan(uint32_t v, uint32_t *wsum, uint32_t &total)
{
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) wsum[w] = x;
  __syncthreads();
  uint32_t base = 0, tot = 0;
  for (int i = 0; i < FAC_THREADS / 32; ++i) { if (i < w) base += wsum[i]; tot += wsum[i]; }
  __syncthreads();
  total = tot;
  return base + x - v;
}

__global__ void __launch_bounds__(FAC_THREADS) k_fac_plan(const SdbFacChan *__restrict__ chans, int C,
                                                          const SdbFacState *__restrict__ state,
                                                          const uint32_t *__restrict__ counts, uint32_t *__restrict__ offs,
                                                          uint32_t *__restrict__ nb_out)
{
  __shared__ uint32_t wsum[FAC_THREADS / 32];
  uint32_t run[SDB_FAC_KINDS] = {0, 0, 0, 0};
  for (int base = 0; base < C; base += FAC_THREADS) {
    const int c = base + threadIdx.x;
    uint32_t n[SDB_FAC_KINDS] = {0, 0, 0, 0};
    if (c < C) {
      const SdbFacChan ch = chans[c];
      const uint32_t nb = (uint32_t) (((unsigned long long) state[c].p + counts[ch.row]) / ch.L);
      nb_out[c] = nb;
      n[0] = ch.L <= 4096 ? nb : 0;
      n[1] = ch.L <= 4096 ? 0 : nb * (ch.L / 4096);
      n[2] = nb * ch.ntiles;
      n[3] = nb ? (ch.L / 2 + FAC_TILE - 1) / FAC_TILE : 0;
    }
#pragma unroll
    for (int k = 0; k < SDB_FAC_KINDS; ++k) {
      uint32_t tot;
      const uint32_t ex = fac_exscan(n[k], wsum, tot);
      if (c < C) offs[k * (C + 1) + c] = run[k] + ex;
      run[k] += tot;
    }
  }
  if (threadIdx.x == 0)
    for (int k = 0; k < SDB_FAC_KINDS; ++k) offs[k * (C + 1) + C] = run[k];
}

// FC.1, L <= 4096: F.2 forward, P = (fma(Xr, Xr, Xi Xi), 0), F.2 inverse, v = |A| for l < L / 2
__global__ void __launch_bounds__(FAC_THREADS) k_fac_small(const SdbFacArgs a)
{
  extern __shared__ float2 sm[];
  const int C = a.n_chans;
  const uint32_t *off = a.offs;
  for (uint32_t u = blockIdx.x; u < off[C]; u += gridDim.x) {
    const int c = fac_find(off, C, u);
    const SdbFacChan ch = a.chans[c];
    const uint32_t j = u - off[c], L = ch.L, p = a.state[c].p;
    const float2 *blk = a.blk + ch.blk_off, *soft = a.soft + (size_t) ch.row * a.sym_cap;
    for (uint32_t i = threadIdx.x; i < L; i += FAC_THREADS) sm[i] = fac_in(blk, soft, j, L, p, i);
    __syncthreads();
    block_fft_inplace<-1, 4>(sm, (int) L, (int) ch.logL, threadIdx.x, FAC_THREADS, ch.tw);
    for (uint32_t i = threadIdx.x; i < L; i += FAC_THREADS)
      sm[i] = make_float2(__fmaf_rn(sm[i].x, sm[i].x, sm[i].y * sm[i].y), 0.0f);
    __syncthreads();
    block_fft_inplace<+1, 4>(sm, (int) L, (int) ch.logL, threadIdx.x, FAC_THREADS, ch.tw);
    float *v = a.work + ch.work_off + (size_t) j * L;
    for (uint32_t i = threadIdx.x; i < L / 2; i += FAC_THREADS) v[i] = d_cabsf(sm[i].x, sm[i].y);
    __syncthreads();
  }
}

// F.3 columns of one 4096-point unit: CW = 4096 / N1 adjacent columns n2, Stockham(N1) over n1, x W_L^(n2 k1) ->
// scr[k1][n2].  SRC 0: the block; SRC 1: the real spectrum P in `work`.
template <int SRC>
__global__ void __launch_bounds__(FAC_THREADS) k_fac_cols(const SdbFacArgs a)
{
  extern __shared__ float2 sm[];
  const int C = a.n_chans;
  const uint32_t *off = a.offs + (C + 1);
  for (uint32_t u = blockIdx.x; u < off[C]; u += gridDim.x) {
    const int c = fac_find(off, C, u);
    const SdbFacChan ch = a.chans[c];
    const uint32_t per = ch.L / 4096, r = u - off[c], j = r / per, g = r - j * per;
    const int N1 = (int) ch.N1, N2 = (int) ch.N2, CW = 4096 / N1, LD = N1 + 1, col0 = (int) g * CW;
    const uint32_t p = a.state[c].p;
    const float2 *blk = a.blk + ch.blk_off, *soft = a.soft + (size_t) ch.row * a.sym_cap;
    const float *wk = a.work + ch.work_off + (size_t) j * ch.L;
    for (int idx = threadIdx.x; idx < 4096; idx += FAC_THREADS) {
      const int rr = idx / CW, cc = idx - rr * CW;
      const uint32_t n = (uint32_t) (rr * N2 + col0 + cc);
      sm[cc * LD + rr] = SRC == 0 ? fac_in(blk, soft, j, ch.L, p, n) : make_float2(wk[n], 0.0f);
    }
    __syncthreads();
    {
      const int per_col = FAC_THREADS / CW, t = threadIdx.x / per_col, lane = threadIdx.x - t * per_col;
      block_fft_inplace<-1, 4>(sm + t * LD, N1, (int) ch.logN1, lane, per_col, ch.twN1);
    }
    float2 *scr = a.scr + ch.scr_off + (size_t) j * ch.L;
    for (int idx = threadIdx.x; idx < 4096; idx += FAC_THREADS) {
      const int k1 = idx / CW, cc = idx - k1 * CW;
      scr[(size_t) k1 * N2 + col0 + cc] = cmul(sm[cc * LD + k1], ldtw(ch.tw, (col0 + cc) * k1));
    }
    __syncthreads();
  }
}

// F.3 rows of one 4096-point unit: RW = 4096 / N2 rows k1, Stockham(N2) over n2 -> X[k1 + N1 k2].  EPI 0: the power
// P[k] = fma(Xr, Xr, Xi Xi) into `work`; EPI 1: v[k] = |X| for k < L / 2 into `work` (P is no longer needed)
template <int EPI>
__global__ void __launch_bounds__(FAC_THREADS) k_fac_rows(const SdbFacArgs a)
{
  extern __shared__ float2 sm[];
  const int C = a.n_chans;
  const uint32_t *off = a.offs + (C + 1);
  for (uint32_t u = blockIdx.x; u < off[C]; u += gridDim.x) {
    const int c = fac_find(off, C, u);
    const SdbFacChan ch = a.chans[c];
    const uint32_t per = ch.L / 4096, r = u - off[c], j = r / per, g = r - j * per;
    const int N1 = (int) ch.N1, N2 = (int) ch.N2, RW = 4096 / N2, LD = N2 + 1, r0 = (int) g * RW;
    const float2 *scr = a.scr + ch.scr_off + (size_t) j * ch.L + (size_t) r0 * N2;
    for (int idx = threadIdx.x; idx < 4096; idx += FAC_THREADS) {
      const int rr = idx / N2, n2 = idx - rr * N2;
      sm[rr * LD + n2] = scr[idx];
    }
    __syncthreads();
    {
      const int per_row = FAC_THREADS / RW, t = threadIdx.x / per_row, lane = threadIdx.x - t * per_row;
      block_fft_inplace<-1, 4>(sm + t * LD, N2, (int) ch.logN2, lane, per_row, ch.twN2);
    }
    float *wk = a.work + ch.work_off + (size_t) j * ch.L;
    const uint32_t half = ch.L / 2;
    for (int idx = threadIdx.x; idx < 4096; idx += FAC_THREADS) {
      const int k2 = idx / RW, rr = idx - k2 * RW;
      const float2 X = sm[rr * LD + k2];
      const uint32_t k = (uint32_t) (r0 + rr + N1 * k2);
      if (EPI == 0) wk[k] = __fmaf_rn(X.x, X.x, X.y * X.y);
      else if (k < half) wk[k] = d_cabsf(X.x, X.y);
    }
    __syncthreads();
  }
}

// the tile of a statistics unit: chain c, block j, lags [lo + FAC_TILE t, min(lo + FAC_TILE (t + 1), hi))
struct FacTileRef { int c; uint32_t j, t, a, n; };
static __device__ __forceinline__ FacTileRef fac_tile(const SdbFacArgs &a, uint32_t u, SdbFacChan &ch)
{
  const int C = a.n_chans;
  const uint32_t *off = a.offs + 2 * (C + 1);
  FacTileRef r;
  r.c = fac_find(off, C, u);
  ch = a.chans[r.c];
  const uint32_t q = u - off[r.c];
  r.j = q / ch.ntiles; r.t = q - r.j * ch.ntiles;
  r.a = ch.lo + r.t * FAC_TILE;
  r.n = min((uint32_t) FAC_TILE, ch.hi - r.a);
  return r;
}

// per tile: the largest v (NaN never counts, as in the tab's `v > max`), the smallest and the first lag of the largest
__global__ void __launch_bounds__(FAC_THREADS) k_fac_tilemax(const SdbFacArgs a)
{
  __shared__ float s_mx[FAC_THREADS / 32], s_mn[FAC_THREADS / 32];
  __shared__ uint32_t s_at[FAC_THREADS / 32];
  const int C = a.n_chans;
  for (uint32_t u = blockIdx.x; u < a.offs[2 * (C + 1) + C]; u += gridDim.x) {
    SdbFacChan ch;
    const FacTileRef r = fac_tile(a, u, ch);
    const float *v = a.work + ch.work_off + (size_t) r.j * ch.L + r.a;
    float mx = -CUDART_INF_F, mn = CUDART_INF_F;
    uint32_t at = 0xffffffffu;
    for (uint32_t i = threadIdx.x; i < r.n; i += FAC_THREADS) {
      const float x = v[i];
      if (x > mx) { mx = x; at = i; }      // ascending i: the first of equal maxima
      mn = fminf(mn, x);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const float omx = __shfl_down_sync(0xffffffffu, mx, o), omn = __shfl_down_sync(0xffffffffu, mn, o);
      const uint32_t oat = __shfl_down_sync(0xffffffffu, at, o);
      if (omx > mx || (omx == mx && oat < at)) { mx = omx; at = oat; }
      mn = fminf(mn, omn);
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { s_mx[w] = mx; s_mn[w] = mn; s_at[w] = at; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int i = 1; i < FAC_THREADS / 32; ++i) {
        if (s_mx[i] > mx || (s_mx[i] == mx && s_at[i] < at)) { mx = s_mx[i]; at = s_at[i]; }
        mn = fminf(mn, s_mn[i]);
      }
      SdbFacTile &T = a.tiles[ch.tile_off + r.j * ch.ntiles + r.t];
      T.max = mx; T.min = mn; T.pos = at == 0xffffffffu ? 0u : r.a + at;
    }
    __syncthreads();
  }
}

// per chain, serially over the feed's tiles in block order: the running maximum entering each tile (FC.2's localMax
// before its first lag), so that every tile finds it in one read
__global__ void k_fac_prefix(const SdbFacArgs a)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.n_chans) return;
  const SdbFacChan ch = a.chans[c];
  SdbFacTile *T = a.tiles + ch.tile_off;
  const uint32_t n = a.nb[c] * ch.ntiles;
  float m = -CUDART_INF_F;
  for (uint32_t i = 0; i < n; ++i) { T[i].pre = m; m = fmaxf(m, T[i].max); }
}

// per tile (FC.2): a value is a record when it exceeds every earlier value of the feed's window (the tiles before it,
// in block order, and the lags before it in the tile); the squares of the others are summed over the 1024 positions of
// the tile by the fixed tree s[i] += s[i + h], h = 512, 256, ..., 1 (binary32, absent positions 0)
__global__ void __launch_bounds__(FAC_THREADS) k_fac_tilepow(const SdbFacArgs a)
{
  __shared__ float s[FAC_TILE];
  __shared__ float s_w[FAC_THREADS / 32];
  __shared__ uint32_t s_cnt;
  const int C = a.n_chans;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (uint32_t u = blockIdx.x; u < a.offs[2 * (C + 1) + C]; u += gridDim.x) {
    SdbFacChan ch;
    const FacTileRef r = fac_tile(a, u, ch);
    // the running maximum entering the tile (k_fac_prefix)
    const float m0 = a.tiles[ch.tile_off + r.j * ch.ntiles + r.t].pre;
    // this thread's four consecutive lags 4 tid .. 4 tid + 3 of the tile
    const float *v = a.work + ch.work_off + (size_t) r.j * ch.L + r.a;
    float x[4];
    float tm = -CUDART_INF_F;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t i = 4 * threadIdx.x + q;
      x[q] = i < r.n ? v[i] : CUDART_NAN_F;
      tm = fmaxf(tm, x[q]);                       // (fmaxf ignores NaN, as `v > max` does)
    }
    // exclusive max-scan of the thread maxima over the CTA
    float incl = tm;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl = fmaxf(incl, y);
    }
    if (lane == 31) s_w[w] = incl;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    float run = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) run = -CUDART_INF_F;
    for (int i = 0; i < w; ++i) run = fmaxf(run, s_w[i]);
    run = fmaxf(run, m0);
    uint32_t cnt = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t i = 4 * threadIdx.x + q;
      float sq = 0.0f;
      if (i < r.n) {
        if (x[q] > run) run = x[q];              // a record: excluded
        else { sq = __fmul_rn(x[q], x[q]); ++cnt; }
      }
      s[i] = sq;
    }
    atomicAdd(&s_cnt, cnt);
    __syncthreads();
    for (int i = threadIdx.x; i < FAC_TILE / 2; i += FAC_THREADS) s[i] = __fadd_rn(s[i], s[i + FAC_TILE / 2]);
    __syncthreads();
    for (int h = FAC_TILE / 4; h > 0; h >>= 1) {
      if ((int) threadIdx.x < h) s[threadIdx.x] = __fadd_rn(s[threadIdx.x], s[threadIdx.x + h]);
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      SdbFacTile &T = a.tiles[ch.tile_off + r.j * ch.ntiles + r.t];
      T.pow = s[0]; T.cnt = s_cnt;
    }
    __syncthreads();
  }
}

// per chain (FC.2 - FC.4), serially over the feed's blocks and their tiles in order
__global__ void k_fac_fixup(const SdbFacArgs a)
{
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= a.n_chans) return;
  const SdbFacChan ch = a.chans[c];
  SdbFacState st = a.state[c];
  const uint32_t nb = a.nb[c];
  float local = -CUDART_INF_F, power = 0.0f;
  uint32_t pos = 0, count = 0;
  for (uint32_t j = 0; j < nb; ++j) {
    float bmax = -CUDART_INF_F, bmin = CUDART_INF_F;
    for (uint32_t t = 0; t < ch.ntiles; ++t) {
      const SdbFacTile T = a.tiles[ch.tile_off + j * ch.ntiles + t];
      if (T.max > local) { local = T.max; pos = T.pos; }
      power = __fadd_rn(power, T.pow);
      count += T.cnt;
      bmax = fmaxf(bmax, T.max); bmin = fminf(bmin, T.min);
    }
    st.max = fmaxf(st.max, bmax); st.min = fminf(st.min, bmin);
    a.slot_max[ch.slot_off + j] = st.max;         // FC.3 divides block j by the maximum including it
  }
  a.state[c].max = st.max; a.state[c].min = st.min;
  sdb_fac_status o;
  o.blocks = nb; o.peak_lag = pos; o.max = st.max; o.min = st.min;
  o.sigmas = 0.0f; o.marker = 0;
  if (nb > 0 && !isinf(local) && count > 0) {
    o.sigmas = __fdiv_rn(local, __fsqrt_rn(__fdiv_rn(power, (float) count)));
    o.marker = (double) o.sigmas > ch.sigma ? 1 : 0;
  }
  a.status[c] = o;
}

// FC.3: fac[l] += alpha (v_j[l] / max_j - fac[l]) for the feed's blocks j in order, 1024 lags per unit
__global__ void __launch_bounds__(FAC_THREADS) k_fac_average(const SdbFacArgs a)
{
  const int C = a.n_chans;
  const uint32_t *off = a.offs + 3 * (C + 1);
  for (uint32_t u = blockIdx.x; u < off[C]; u += gridDim.x) {
    const int c = fac_find(off, C, u);
    const SdbFacChan ch = a.chans[c];
    const uint32_t nb = a.nb[c], half = ch.L / 2, l0 = (u - off[c]) * FAC_TILE;
    float *fac = a.fac + ch.fac_off;
    for (uint32_t l = l0 + threadIdx.x; l < min(l0 + FAC_TILE, half); l += FAC_THREADS) {
      float f = fac[l];
      for (uint32_t j = 0; j < nb; ++j) {
        const float t = __fdiv_rn(a.work[ch.work_off + (size_t) j * ch.L + l], a.slot_max[ch.slot_off + j]);
        f = __fadd_rn(f, __fmul_rn(ch.alpha, __fsub_rn(t, f)));
      }
      fac[l] = f;
    }
  }
}

// the feed's symbols past its last completed block become the carried block; one CTA per chain
__global__ void __launch_bounds__(FAC_THREADS) k_fac_tail(const SdbFacArgs a)
{
  const int c = blockIdx.x;
  const SdbFacChan ch = a.chans[c];
  const uint32_t n = a.counts[ch.row], p = a.state[c].p, tot = p + n, nb = tot / ch.L, rem = tot - nb * ch.L;
  const float2 *soft = a.soft + (size_t) ch.row * a.sym_cap;
  float2 *blk = a.blk + ch.blk_off;
  if (nb == 0) for (uint32_t i = threadIdx.x; i < n; i += FAC_THREADS) blk[p + i] = soft[i];
  else         for (uint32_t i = threadIdx.x; i < rem; i += FAC_THREADS) blk[i] = soft[nb * ch.L - p + i];
  __syncthreads();
  if (threadIdx.x == 0) a.state[c].p = rem;
}

cudaError_t sdb_launch_fac(const SdbLaunchCtx &c, const SdbFacArgs &a, const int grid[SDB_FAC_KINDS])
{
  if (a.n_chans <= 0) return cudaSuccess;
  auto count = [&]() { if (c.launch_counter) ++*c.launch_counter; };
  // shared memory: the block (F.2), or 4096 points of columns / rows with one padding element per column / row
  const size_t smem_small = (size_t) 4096 * sizeof(float2), smem_pass = (size_t) (4096 + 64) * sizeof(float2);
  k_fac_plan<<<1, FAC_THREADS, 0, c.stream>>>(a.chans, a.n_chans, a.state, a.counts, a.offs, a.nb); count();
  if (grid[0]) { k_fac_small<<<grid[0], FAC_THREADS, smem_small, c.stream>>>(a); count(); }
  if (grid[1]) {
    k_fac_cols<0><<<grid[1], FAC_THREADS, smem_pass, c.stream>>>(a); count();
    k_fac_rows<0><<<grid[1], FAC_THREADS, smem_pass, c.stream>>>(a); count();
    k_fac_cols<1><<<grid[1], FAC_THREADS, smem_pass, c.stream>>>(a); count();
    k_fac_rows<1><<<grid[1], FAC_THREADS, smem_pass, c.stream>>>(a); count();
  }
  k_fac_tilemax<<<grid[2], FAC_THREADS, 0, c.stream>>>(a); count();
  k_fac_prefix<<<(a.n_chans + 127) / 128, 128, 0, c.stream>>>(a); count();
  k_fac_tilepow<<<grid[2], FAC_THREADS, 0, c.stream>>>(a); count();
  k_fac_fixup<<<(a.n_chans + 127) / 128, 128, 0, c.stream>>>(a); count();
  k_fac_average<<<grid[3], FAC_THREADS, 0, c.stream>>>(a); count();
  k_fac_tail<<<a.n_chans, FAC_THREADS, 0, c.stream>>>(a); count();
  return cudaGetLastError();
}
