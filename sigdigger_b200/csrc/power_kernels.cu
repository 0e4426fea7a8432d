// power_kernels.cu -- the "power" inspector (SPEC PW, oracle/SPEC_PW.md): the RMS tool's integrated channel power
// (Default/RMSInspector/RMSInspector.cpp).  Per channel sample p = re re + im im in binary32 (two rounded products,
// one rounded add), widened to binary64 and added with Kahan compensation (RMSInspector.cpp:551-556); once a group
// holds M samples its mean acc / n, rounded to binary32, is one output sample (mean, 0) with hard symbol 0
// (:329-336).  The group (acc, c, n) carries across feeds.
//
// The recurrence is serial, so each lane owns one chain (one power channel of one stream) and a warp 32 of them.  The
// warp stages 32 consecutive samples of each of its chains through a 32 x 33 shared-memory tile: one chain's samples
// are one coalesced 256-byte load, and the padded column a lane then walks is free of bank conflicts.  The 32 row
// loads of the next chunk are issued together, into registers, before the lane runs the Kahan steps of the current
// chunk, so the HBM round trip overlaps the dependent binary64 adds instead of preceding each row.  acc, c and n stay
// in registers for the whole feed.  Built with -fmad=false; the binary64 steps are written with round-to-nearest
// intrinsics so that no step is contracted or reordered.
#include "sdb_internal.h"

__global__ void __launch_bounds__(32) k_power_integrate(const SdbPowerChain *__restrict__ chains, int n_chains,
                                                        const float2 *__restrict__ chan_in, uint32_t n_hops,
                                                        SdbPowerCarry *__restrict__ carry, float2 *__restrict__ soft,
                                                        unsigned char *__restrict__ hard,
                                                        uint32_t *__restrict__ sym_counts, size_t sym_cap)
{
  __shared__ float tile[32][33];                       // [chain of the warp][sample of the chunk]
  __shared__ size_t s_off[32];
  __shared__ unsigned long long s_len[32];
  const int lane = threadIdx.x;
  const int me = blockIdx.x * 32 + lane;
  const bool valid = me < n_chains;
  SdbPowerChain ch{};
  SdbPowerCarry st{ 0.0, 0.0, 0ull };
  if (valid) { ch = chains[me]; st = carry[ch.out]; }
  const unsigned long long len = valid ? (unsigned long long) n_hops * ch.halfsz : 0ull;
  s_off[lane] = ch.in_off; s_len[lane] = len;          // (a lane without a chain reads chan_in[0] and discards it)
  unsigned long long len_max = len;
  for (int o = 16; o; o >>= 1) len_max = max(len_max, __shfl_xor_sync(0xffffffffu, len_max, o));
  __syncwarp();
  // samples c0 + lane of every chain of the warp; past a chain's end the index is clamped and the value discarded
  float2 v[32];
  auto load_rows = [&](unsigned long long c0) {
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const unsigned long long l = s_len[j], i = c0 + lane;
      v[j] = __ldg(chan_in + s_off[j] + (i < l ? i : (l ? l - 1 : 0)));
    }
  };
  if (len_max) load_rows(0);
  double acc = st.acc, c = st.c;
  unsigned long long n = st.n;
  const unsigned long long M = ch.M;
  float2 *so = soft + (size_t) (valid ? ch.out : 0) * sym_cap;
  unsigned char *ho = hard + (size_t) (valid ? ch.out : 0) * sym_cap;
  uint32_t nout = 0;
  for (unsigned long long c0 = 0; c0 < len_max; c0 += 32) {
    // row j: samples c0 .. c0 + 31 of chain j of the warp, as powers
#pragma unroll
    for (int j = 0; j < 32; ++j)
      tile[j][lane] = c0 + lane < s_len[j] ? __fadd_rn(__fmul_rn(v[j].x, v[j].x), __fmul_rn(v[j].y, v[j].y)) : 0.0f;
    __syncwarp();
    if (c0 + 32 < len_max) load_rows(c0 + 32);         // in flight during the Kahan steps below
    const int take = len > c0 ? (int) min(32ull, len - c0) : 0;
    for (int i = 0; i < take; ++i) {
      const double y = __dsub_rn((double) tile[lane][i], c);
      const double t = __dadd_rn(acc, y);
      c = __dsub_rn(__dsub_rn(t, acc), y);
      acc = t;
      if (++n >= M) {
        so[nout] = make_float2(__double2float_rn(__ddiv_rn(acc, (double) n)), 0.0f);
        ho[nout] = 0;
        ++nout;
        acc = c = 0.0; n = 0;
      }
    }
    __syncwarp();
  }
  if (valid) {
    carry[ch.out] = SdbPowerCarry{ acc, c, n };
    sym_counts[ch.out] = nout;
  }
}

cudaError_t sdb_launch_power_integrate(const SdbLaunchCtx &c, const SdbPowerChain *chains, int n_chains,
                                       const float2 *chan_in, uint32_t n_hops, SdbPowerCarry *carry, float2 *soft,
                                       uint8_t *hard, uint32_t *sym_counts, size_t sym_cap)
{
  if (n_chains <= 0) return cudaSuccess;
  // one warp per CTA: the work is a latency-bound recurrence per lane, best spread over as many SMs as there are warps
  k_power_integrate<<<(n_chains + 31) / 32, 32, 0, c.stream>>>(chains, n_chains, chan_in, n_hops, carry, soft, hard,
                                                               sym_counts, sym_cap);
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}

// Offline power integration of `batch` captured channel-rate buffers (the RMS tab's raw mode over a capture): one
// chain per buffer, each starting an empty group, through the kernel the engine runs.
extern "C" long sdb_task_power(const sdb_complex *src, size_t n, size_t batch, uint64_t integrate_samples,
                               sdb_complex *means, uint32_t *counts, size_t cap)
{
  if (!src || !means || !counts || n == 0 || batch == 0) return fail("invalid argument");
  if (n > UINT32_MAX || batch > (size_t) INT32_MAX) return fail("power task: buffer too long or batch too large");
  const uint64_t M = integrate_samples ? integrate_samples : 1;
  if (cap < n / M) return fail("power task: cap must hold n / integrate_samples means");
  if (sdb_device_count() <= 0) return fail("no CUDA device: sigdigger_b200 has no CPU fallback");
  std::vector<SdbPowerChain> pw(batch);
  for (size_t b = 0; b < batch; ++b) pw[b] = SdbPowerChain{ b * n, (uint32_t) n, (uint32_t) b, M };
  const size_t rows = std::max<size_t>(cap, 1);
  DevBuf<float2> d_src, d_soft; DevBuf<uint8_t> d_hard; DevBuf<uint32_t> d_cnt;
  DevBuf<SdbPowerChain> d_pw; DevBuf<SdbPowerCarry> d_carry;
  CK(d_src.alloc(n * batch)); CK(d_soft.alloc(rows * batch)); CK(d_hard.alloc(rows * batch)); CK(d_cnt.alloc(batch));
  CK(d_pw.alloc(batch)); CK(d_carry.alloc(batch));
  CK(cudaMemcpy(d_src, src, n * batch * sizeof(float2), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(d_pw, pw.data(), batch * sizeof(SdbPowerChain), cudaMemcpyHostToDevice));
  CK(cudaMemset(d_carry, 0, batch * sizeof(SdbPowerCarry)));
  SdbLaunchCtx ctx{ 0, nullptr };
  // every buffer is one hop of n samples
  CK(sdb_launch_power_integrate(ctx, d_pw, (int) batch, d_src, 1, d_carry, d_soft, d_hard, d_cnt, rows));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(counts, d_cnt, batch * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  if (cap) CK(cudaMemcpy(means, d_soft, cap * batch * sizeof(float2), cudaMemcpyDeviceToHost));
  return 0;
}
