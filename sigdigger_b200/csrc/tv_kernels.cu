// tv_kernels.cu -- analog-TV processor of the inspector's TV tab on the GPU (SURVEY.md 8(f) rank 4; SPEC.md TV).
//
// Replaces, for a batch of processors, what the reference runs per TV tab on a worker thread:
//   TVProcessorTab::feed          Default/GenericInspector/TVProcessorTab.cpp:601-620   k |x| + dc  /  k arg(x)/pi + dc
//   TVProcessorWorker::work       Default/GenericInspector/TVProcessorWorker.cpp:120-151 su_tv_processor_feed per sample,
//                                                                                       take_frame on a completed frame
//   start / setParams             TVProcessorWorker.cpp:186-239                          su_tv_processor_new / _set_params
// The processor is a per-sample recurrence (flywheel sync separator + raster), so one stream cannot be split:
// ONE WARP PER PROCESSOR.  Lane 0 runs the step of sdb_tv_steps.h with the loop state in registers, the comb delay
// line and the row being drawn in shared memory; the warp loads the input 32 samples at a time (coalesced) and hands
// them to lane 0 by shuffle, and all 32 lanes store a finished row into the frame ring (coalesced) and clear it.
// Bound: serial latency of the step (one processor advances a few MS/s; a batch scales with the SM count).
// k_tv_insp runs the same warp over an engine inspector's device-side soft symbols: the inspector panel's Analog TV
// tab (InspectorUI.cpp:851-852, oracle/SPEC_TI.md), one processor per (TV channel, stream), launched by engine.cu.
// Compiled with -fmad=false: bit-identical to oracle/tvproc.c and to the host step of <sigutils/tvproc.h>.
#include "sdb_tv_steps.h"
#include <vector>
#include <string.h>

__global__ void __launch_bounds__(32) k_tv_feed(const SdbTvCfg c, SdbTvState *__restrict__ states,
                                                float *__restrict__ delays, float *__restrict__ lines,
                                                float *__restrict__ rings, const float *__restrict__ x, size_t stride,
                                                size_t n, unsigned *__restrict__ frames_done)
{
  extern __shared__ float s_tv[];                // [W] row being drawn | [delay_len] comb delay line
  float *s_line = s_tv, *s_delay = s_tv + c.W;
  const int b = blockIdx.x, lane = threadIdx.x;
  float *g_line = lines + (size_t) b * c.W, *g_delay = delays + (size_t) b * c.delay_len;
  float *ring = rings + (size_t) b * SDB_TV_RING * c.H * c.W;
  for (int k = lane; k < c.W; k += 32) s_line[k] = g_line[k];
  for (int k = lane; k < c.delay_len; k += 32) s_delay[k] = g_delay[k];
  SdbTvState st;
  if (lane == 0) st = states[b];
  __syncwarp();
  const float *__restrict__ xs = x + (size_t) b * stride;
  unsigned done = 0;
  for (size_t i0 = 0; i0 < n; i0 += 32) {
    const float xv = i0 + lane < n ? __ldg(xs + i0 + lane) : 0.0f;
    const int cnt = n - i0 < 32 ? (int) (n - i0) : 32;
    for (int j = 0; j < cnt; ++j) {
      const float xj = __shfl_sync(0xffffffffu, xv, j);
      int flags = 0, frow = -1, fslot = 0;
      if (lane == 0) flags = sdb_tv_step(c, st, s_delay, s_line, xj, &frow, &fslot);
      flags = __shfl_sync(0xffffffffu, flags, 0);
      if (flags & SDB_TV_LINE_DONE) {
        frow = __shfl_sync(0xffffffffu, frow, 0);
        fslot = __shfl_sync(0xffffffffu, fslot, 0);
        if (frow >= 0) {
          float *__restrict__ dst = ring + ((size_t) fslot * c.H + frow) * c.W;
          for (int k = lane; k < c.W; k += 32) dst[k] = s_line[k];
        }
        for (int k = lane; k < c.W; k += 32) s_line[k] = 0.0f;
        __syncwarp();
        if (flags & SDB_TV_FRAME_DONE) ++done;
      }
    }
  }
  __syncwarp();
  for (int k = lane; k < c.W; k += 32) g_line[k] = s_line[k];
  for (int k = lane; k < c.delay_len; k += 32) g_delay[k] = s_delay[k];
  if (lane == 0) { states[b] = st; frames_done[b] = done; }
}

// TVProcessorTab::feed: mode 0 = Decider::MODULUS, 1 = ARGUMENT (SPEC M elementary functions)
__global__ void k_tv_feed_transform(const float2 *__restrict__ x, size_t n, int mode, float k, float dc,
                                    float *__restrict__ out)
{
  const size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float2 v = x[i];
  out[i] = mode == 0 ? k * sqrtf(v.x * v.x + v.y * v.y) + dc
                     : k * d_atan2f(v.y, v.x) / 3.14159265358979323846f + dc;
}

// The engine's Analog TV tab (oracle/SPEC_TI.md): one warp per (TV channel, stream), grid (n_streams, n_chans), on
// the inspector stream after the feed's chains.  As k_tv_feed, but the input is the row's soft symbols and their
// device-side count, converted in the coalesced load with k_tv_feed_transform's expression (TI.1), and the feed's
// first completed frame is copied from its ring slot to the posted frame as soon as it completes (TI.3: four more
// frames of the same feed would overwrite the slot).  Dynamic shared memory: the largest W + delay_len.
__global__ void __launch_bounds__(32) k_tv_insp(const SdbTvInspChan *__restrict__ chans, int n_channels,
                                                const float2 *__restrict__ soft, const uint32_t *__restrict__ counts,
                                                size_t sym_cap, SdbTvState *__restrict__ states,
                                                float *__restrict__ delays, float *__restrict__ lines,
                                                float *__restrict__ rings, float *__restrict__ posts,
                                                sdb_tv_status *__restrict__ status)
{
  const SdbTvInspChan &ch = chans[blockIdx.y];
  const int s = blockIdx.x, lane = threadIdx.x;
  const unsigned p = ch.chain0 + s;
  const size_t row = (size_t) s * n_channels + ch.k;
  const unsigned n = counts[row];
  if (n == 0) {                                    // TI.2: nothing changes
    if (lane == 0) status[p].completed = 0;
    return;
  }
  const SdbTvCfg c = ch.c;
  const int mode = ch.mode;
  const float gain = ch.gain, dc = ch.dc;
  extern __shared__ float s_tv[];                  // [W] row being drawn | [delay_len] comb delay line
  float *s_line = s_tv, *s_delay = s_tv + c.W;
  const size_t px = (size_t) c.H * c.W;
  float *g_line = lines + ch.line_off + (size_t) s * c.W, *g_delay = delays + ch.delay_off + (size_t) s * c.delay_len;
  float *ring = rings + ch.ring_off + (size_t) s * SDB_TV_RING * px;
  float *__restrict__ post = posts + ch.post_off + (size_t) s * px;
  for (int k = lane; k < c.W; k += 32) s_line[k] = g_line[k];
  for (int k = lane; k < c.delay_len; k += 32) s_delay[k] = g_delay[k];
  SdbTvState st;
  if (lane == 0) st = states[p];
  __syncwarp();
  const float2 *__restrict__ xs = soft + row * sym_cap;
  unsigned done = 0;
  for (unsigned i0 = 0; i0 < n; i0 += 32) {
    float xv = 0.0f;
    if (i0 + lane < n) {
      const float2 v = xs[i0 + lane];
      xv = mode == 0 ? gain * sqrtf(v.x * v.x + v.y * v.y) + dc
                     : gain * d_atan2f(v.y, v.x) / 3.14159265358979323846f + dc;
    }
    const int cnt = n - i0 < 32 ? (int) (n - i0) : 32;
    for (int j = 0; j < cnt; ++j) {
      const float xj = __shfl_sync(0xffffffffu, xv, j);
      int flags = 0, frow = -1, fslot = 0;
      if (lane == 0) flags = sdb_tv_step(c, st, s_delay, s_line, xj, &frow, &fslot);
      flags = __shfl_sync(0xffffffffu, flags, 0);
      if (flags & SDB_TV_LINE_DONE) {
        frow = __shfl_sync(0xffffffffu, frow, 0);
        fslot = __shfl_sync(0xffffffffu, fslot, 0);
        float *__restrict__ slot = ring + (size_t) fslot * px;
        if (frow >= 0)
          for (int k = lane; k < c.W; k += 32) slot[(size_t) frow * c.W + k] = s_line[k];
        for (int k = lane; k < c.W; k += 32) s_line[k] = 0.0f;
        __syncwarp();
        if ((flags & SDB_TV_FRAME_DONE) && ++done == 1) {
          for (size_t k = lane; k < px; k += 32) post[k] = slot[k];
          __syncwarp();
        }
      }
    }
  }
  __syncwarp();
  for (int k = lane; k < c.W; k += 32) g_line[k] = s_line[k];
  for (int k = lane; k < c.delay_len; k += 32) g_delay[k] = s_delay[k];
  if (lane == 0) {
    states[p] = st;
    sdb_tv_status o = status[p];
    if (done) o.posted_no = st.frames - done + 1;
    o.frames = st.frames; o.completed = done; o.width = (uint32_t) c.W; o.height = (uint32_t) c.H;
    o.line_len = st.est_line_len; o.hsync_len = st.est_hsync_len; o.agc_gain = st.agc_gain;
    status[p] = o;
  }
}

cudaError_t sdb_launch_tv_insp(const SdbLaunchCtx &ctx, const SdbTvInspArgs &a)
{
  if (a.n_chans <= 0) return cudaSuccess;
  k_tv_insp<<<dim3((unsigned) a.n_streams, (unsigned) a.n_chans), 32, a.smem, ctx.stream>>>(
      a.chans, a.n_channels, a.soft, a.counts, a.sym_cap, a.state, a.delay, a.line, a.ring, a.post, a.status);
  if (ctx.launch_counter) ++*ctx.launch_counter;
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
struct sdb_tv_processor {
  int device = 0; unsigned batch = 0;
  sdb_tv_params prm; SdbTvCfg cfg;
  DevBuf<SdbTvState> d_state; DevBuf<float> d_delay, d_line, d_ring, d_x; DevBuf<unsigned> d_done;
  Stream stream;
};

extern "C" void sdb_tv_params_pal(sdb_tv_params *p, float samp_rate) { if (p) sdb_tv_preset(*p, samp_rate, true); }
extern "C" void sdb_tv_params_ntsc(sdb_tv_params *p, float samp_rate) { if (p) sdb_tv_preset(*p, samp_rate, false); }

extern "C" void sdb_tv_processor_destroy(sdb_tv_processor_t *t)
{
  if (!t) return;
  cudaSetDevice(t->device);
  if (t->stream) cudaStreamSynchronize(t->stream);
  delete t;
}

// su_tv_processor_new (TVProcessorWorker.cpp:204): NULL on invalid parameters ("sample rate / baud rate sufficiently
// high", :206) -- and, here, without a CUDA device (no CPU fallback)
extern "C" sdb_tv_processor_t *sdb_tv_processor_new(const sdb_tv_params *p, uint32_t batch, int device)
{
  if (!p || batch < 1) { fail("invalid arguments"); return nullptr; }
  if (sdb_device_count() <= 0) { fail("no CUDA device: sigdigger_b200 has no CPU fallback"); return nullptr; }
  if (!sdb_tv_params_valid(*p)) { fail("TV processor: invalid parameters"); return nullptr; }
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); fail("cudaSetDevice failed"); return nullptr; }
  sdb_tv_processor *t = new sdb_tv_processor();
  t->device = device; t->batch = batch; t->prm = *p;
  sdb_tv_derive(*p, t->cfg);
  const SdbTvCfg &c = t->cfg;
  const size_t B = batch;
  bool ok = t->d_state.alloc(B) == cudaSuccess && t->d_delay.alloc(B * c.delay_len) == cudaSuccess &&
            t->d_line.alloc(B * c.W) == cudaSuccess && t->d_ring.alloc(B * SDB_TV_RING * c.H * c.W) == cudaSuccess &&
            t->d_done.alloc(B) == cudaSuccess &&
            t->stream.create(cudaStreamNonBlocking) == cudaSuccess;
  if (ok) {
    SdbTvState s0; sdb_tv_state_init(c, s0);
    std::vector<SdbTvState> h(B, s0);
    ok = cudaMemcpy(t->d_state, h.data(), B * sizeof(SdbTvState), cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemset(t->d_delay, 0, B * c.delay_len * sizeof(float)) == cudaSuccess &&
         cudaMemset(t->d_line, 0, B * c.W * sizeof(float)) == cudaSuccess &&
         cudaMemset(t->d_ring, 0, B * SDB_TV_RING * c.H * c.W * sizeof(float)) == cudaSuccess;
  }
  if (!ok) { cudaGetLastError(); fail("out of device memory (TV processor)"); sdb_tv_processor_destroy(t); return nullptr; }
  return t;
}

// su_tv_processor_set_params (TVProcessorWorker.cpp:222): the picture geometry is fixed at creation, everything else
// (tolerances, time constants, sync / AGC / comb switches, pulse lengths) takes effect at the next sample
extern "C" int sdb_tv_processor_set_params(sdb_tv_processor_t *t, const sdb_tv_params *p)
{
  if (!t || !p) return fail("null argument");
  if (!sdb_tv_params_valid(*p)) return fail("TV processor: invalid parameters");
  SdbTvCfg c; sdb_tv_derive(*p, c);
  if (c.W != t->cfg.W || c.delay_len != t->cfg.delay_len || c.H != t->cfg.H || c.interlace != t->cfg.interlace)
    return fail("TV processor: picture geometry cannot change while running");
  CK(cudaSetDevice(t->device));
  CK(cudaStreamSynchronize(t->stream));
  t->prm = *p; t->cfg = c;
  return 0;
}

extern "C" int sdb_tv_processor_geometry(const sdb_tv_processor_t *t, uint32_t *width, uint32_t *height)
{
  if (!t) return fail("null argument");
  if (width) *width = (uint32_t) t->cfg.W;
  if (height) *height = (uint32_t) t->cfg.H;
  return 0;
}

static long tv_feed(sdb_tv_processor *t, const float *x_dev, size_t stride, size_t n, uint32_t *frames_done)
{
  const SdbTvCfg &c = t->cfg;
  const size_t smem = (size_t) (c.W + c.delay_len) * sizeof(float);
  k_tv_feed<<<t->batch, 32, smem, t->stream>>>(c, t->d_state, t->d_delay, t->d_line, t->d_ring, x_dev, stride, n,
                                               t->d_done);
  CK(cudaGetLastError());
  std::vector<unsigned> h(t->batch);
  CK(cudaMemcpyAsync(h.data(), t->d_done, t->batch * sizeof(unsigned), cudaMemcpyDeviceToHost, t->stream));
  CK(cudaStreamSynchronize(t->stream));
  long total = 0;
  for (unsigned b = 0; b < t->batch; ++b) { if (frames_done) frames_done[b] = h[b]; total += h[b]; }
  return total;
}

// TVProcessorWorker::work over a batch: x[batch][stride] host floats, n per processor; frames_done[batch] (may be NULL).
// Returns the number of frames completed in this call over the batch.
extern "C" long sdb_tv_processor_feed(sdb_tv_processor_t *t, const float *x, size_t stride, size_t n, uint32_t *frames_done)
{
  if (!t || !x) return fail("null argument");
  if (n == 0) return 0;
  if (stride < n) return fail("stride < n");
  CK(cudaSetDevice(t->device));
  const size_t need = (size_t) t->batch * n;
  if (t->d_x.size() < need) {
    CK(cudaStreamSynchronize(t->stream));
    CK(t->d_x.alloc(need));
  }
  CK(cudaMemcpy2DAsync(t->d_x, n * sizeof(float), x, stride * sizeof(float), n * sizeof(float), t->batch,
                        cudaMemcpyHostToDevice, t->stream));
  return tv_feed(t, t->d_x, n, n, frames_done);
}

extern "C" long sdb_tv_processor_feed_device(sdb_tv_processor_t *t, const float *x_dev, size_t stride, size_t n,
                                             uint32_t *frames_done)
{
  if (!t || !x_dev) return fail("null argument");
  if (n == 0) return 0;
  if (stride < n) return fail("stride < n");
  CK(cudaSetDevice(t->device));
  return tv_feed(t, x_dev, stride, n, frames_done);
}

extern "C" int sdb_tv_processor_frames(sdb_tv_processor_t *t, uint64_t *counts)
{
  if (!t || !counts) return fail("null argument");
  CK(cudaSetDevice(t->device));
  std::vector<SdbTvState> h(t->batch);
  CK(cudaMemcpy(h.data(), t->d_state, t->batch * sizeof(SdbTvState), cudaMemcpyDeviceToHost));
  for (unsigned b = 0; b < t->batch; ++b) counts[b] = h[b].frames;
  return 0;
}

// su_tv_processor_take_frame (TVProcessorWorker.cpp:143): frame `frame_no` (0-based count of completed frames) of
// processor `which`, while it is still in the ring (the last SDB_TV_RING - 1 completed frames; frame_no == frames
// reads the picture in progress)
extern "C" int sdb_tv_processor_read_frame(sdb_tv_processor_t *t, uint32_t which, uint64_t frame_no, float *out, size_t cap)
{
  if (!t || !out || which >= t->batch) return fail("invalid argument");
  const size_t px = (size_t) t->cfg.W * t->cfg.H;
  if (cap < px) return fail("destination too small");
  CK(cudaSetDevice(t->device));
  SdbTvState s;
  CK(cudaMemcpy(&s, t->d_state + which, sizeof(s), cudaMemcpyDeviceToHost));
  if (frame_no > s.frames || frame_no + SDB_TV_RING <= s.frames) return fail("frame no longer (or not yet) in the ring");
  CK(cudaMemcpy(out, t->d_ring + ((size_t) which * SDB_TV_RING + frame_no % SDB_TV_RING) * px, px * sizeof(float),
                 cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int sdb_tv_processor_estimates(sdb_tv_processor_t *t, uint32_t which, float *line_len, float *hsync_len, float *gain)
{
  if (!t || which >= t->batch) return fail("invalid argument");
  CK(cudaSetDevice(t->device));
  SdbTvState s;
  CK(cudaMemcpy(&s, t->d_state + which, sizeof(s), cudaMemcpyDeviceToHost));
  if (line_len) *line_len = s.est_line_len;
  if (hsync_len) *hsync_len = s.est_hsync_len;
  if (gain) *gain = s.agc_gain;
  return 0;
}

extern "C" int sdb_tv_feed_transform(const sdb_complex *x, size_t n, int mode, float k, float dc, float *out)
{
  if (!x || !out) return fail("null argument");
  if (mode != 0 && mode != 1) return fail("mode: 0 modulus, 1 argument");
  if (sdb_device_count() <= 0) return fail("no CUDA device: sigdigger_b200 has no CPU fallback");
  if (n == 0) return 0;
  DevBuf<float2> dx; DevBuf<float> dout;
  CK(dx.alloc(n));
  if (dout.alloc(n) != cudaSuccess) return fail("out of device memory");
  cudaError_t e = cudaMemcpy(dx, x, n * sizeof(float2), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    k_tv_feed_transform<<<(unsigned) ((n + 255) / 256), 256>>>(dx, n, mode, k, dc, dout);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(out, dout, n * sizeof(float), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(cudaGetErrorString(e));
  return 0;
}
