// spectsched_kernels.cu -- scheduled inspector spectra and baud estimates (oracle/SPEC_US.md).
//
// A scheduled channel emits at t_j = j I channel samples since it started, with a frame of the Ns + 1 samples
// c[t_j - Ns - 1 .. t_j - 1], wherever they lie relative to feed boundaries.  The samples a future frame can still
// need live in a per-(channel, stream) ring of Ns + 1 entries indexed by t mod (Ns + 1).  Per feed, on the inspector
// stream:
//   k_spectsched_gather  assembles each emission's frame contiguously, from the ring and from the feed's channel
//                        stream, and marks its emission slot in the per-slot channel table as one full frame
//                        (halfsz = Ns + 1) or as empty (halfsz = 0);
//   k_spectsrc           (fft_kernels.cu, unchanged) transforms every slot as a feed of one hop of Ns + 1 samples;
//   k_spectsched_ring    writes the feed's samples that a later frame can still need into the ring.
// The gather runs before the ring update of the same feed: a later emission of the feed may overwrite ring entries
// an earlier one reads.  Both are copies; the host computes the schedule (every stream of a feed produces the same
// number of channel samples).
#include "sdb_internal.h"

// one CTA per (emission slot, stream)
__global__ void __launch_bounds__(256) k_spectsched_gather(const SdbSchedChan *__restrict__ sched,
                                                           const int *__restrict__ slot_chan,
                                                           SdbChannelDev *__restrict__ slot_dev,
                                                           const float2 *__restrict__ chan_in, size_t chan_stride,
                                                           const float2 *__restrict__ ring, size_t ring_stride,
                                                           float2 *__restrict__ frames, size_t frame_stride)
{
  const int slot = blockIdx.x, st = blockIdx.y;
  const SdbSchedChan c = sched[slot_chan[slot]];
  const uint32_t e = (uint32_t) slot - c.slot0;
  if (st == 0 && threadIdx.x == 0) slot_dev[slot].halfsz = e < c.n_emit ? (int) c.ns1 : 0;
  if (e >= c.n_emit) return;
  const unsigned long long m0 = c.t_first + (unsigned long long) e * c.interval - c.ns1;   // first sample of the frame
  const uint32_t r0 = (uint32_t) (m0 % c.ns1);
  const float2 *__restrict__ in = chan_in + (size_t) st * chan_stride + c.in_off;
  const float2 *__restrict__ rg = ring + (size_t) st * ring_stride + c.ring_off;
  float2 *__restrict__ out = frames + (size_t) st * frame_stride + c.frame_off + (size_t) e * c.ns1;
  for (uint32_t i = threadIdx.x; i < c.ns1; i += blockDim.x) {
    const unsigned long long m = m0 + i;
    uint32_t r = r0 + i;
    if (r >= c.ns1) r -= c.ns1;
    out[i] = m >= c.t0 ? in[m - c.t0] : rg[r];
  }
}

// one CTA per (scheduled channel, stream): feed samples [w_from, w_to) -> ring entries (t0 + i) mod (Ns + 1)
__global__ void __launch_bounds__(256) k_spectsched_ring(const SdbSchedChan *__restrict__ sched,
                                                         const float2 *__restrict__ chan_in, size_t chan_stride,
                                                         float2 *__restrict__ ring, size_t ring_stride)
{
  const SdbSchedChan c = sched[blockIdx.x];
  const int st = blockIdx.y;
  if (c.w_to <= c.w_from) return;
  const uint32_t n = c.w_to - c.w_from, r0 = (uint32_t) ((c.t0 + c.w_from) % c.ns1);   // n <= Ns + 1
  const float2 *__restrict__ in = chan_in + (size_t) st * chan_stride + c.in_off + c.w_from;
  float2 *__restrict__ rg = ring + (size_t) st * ring_stride + c.ring_off;
  for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
    uint32_t r = r0 + i;
    if (r >= c.ns1) r -= c.ns1;
    rg[r] = in[i];
  }
}

cudaError_t sdb_launch_spectsched_gather(const SdbLaunchCtx &c, const SdbSchedChan *sched, const int *slot_chan,
                                         SdbChannelDev *slot_dev, int n_slots, int n_streams, const float2 *chan_in,
                                         size_t chan_stride, const float2 *ring, size_t ring_stride, float2 *frames,
                                         size_t frame_stride)
{
  k_spectsched_gather<<<dim3(n_slots, n_streams), 256, 0, c.stream>>>(sched, slot_chan, slot_dev, chan_in, chan_stride,
                                                                      ring, ring_stride, frames, frame_stride);
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}

cudaError_t sdb_launch_spectsched_ring(const SdbLaunchCtx &c, const SdbSchedChan *sched, int n_sched, int n_streams,
                                       const float2 *chan_in, size_t chan_stride, float2 *ring, size_t ring_stride)
{
  k_spectsched_ring<<<dim3(n_sched, n_streams), 256, 0, c.stream>>>(sched, chan_in, chan_stride, ring, ring_stride);
  if (c.launch_counter) ++*c.launch_counter;
  return cudaGetLastError();
}
