// panoramic.cu -- the panoramic scanner's sweep behind the C-ABI (BASELINE.json configs[4]; SURVEY.md 8(e)).
//
// What the reference does on the GUI thread per PSD message of a wide-spectrum analyzer
// (Panoramic/Scanner.cpp:503-523: view.feed(psd, nullptr, fftSize, fc); constructor / hop plan :296-372), spread over
// the GPUs of one node, one process per GPU:
//
//     rank r : hops [lo_r, hi_r)  --PSD (engine)-->  SpectrumView projection  --contribution lists--+
//                                  `-> per-hop channel detector (optional)                          | gather to rank 0
//     rank 0 : accumulate(all contribution lists, in global hop order) + gap fill  <----------------+ (NCCL, NVLink)
//
// Per-bin state of the SpectrumView depends only on that bin's own contributions in hop order (SPEC V), so applying
// the gathered lists in rank order (= hop order: shards are contiguous) reproduces the reference's sequential
// feed() value by value.  This gather is the ONLY collective on the path (the PSDs never move): every rank packs
// {j0, nb, va, vc (, channel lists)} of its shard into one device buffer and rank 0 posts one ncclRecv per peer
// inside a group (ncclSend on the peers).  NCCL is bound at run time (dlopen "libnccl.so.2": the process that
// initialised torch.distributed has it loaded already); a single rank needs no NCCL at all.
#include "sdb_internal.h"
#include <nccl.h>
#include <dlfcn.h>

#include <algorithm>
#include <string>
#include <vector>
#include <string.h>
#include <stdlib.h>

static thread_local std::string g_perr;
static int pfail(const std::string &m) { g_perr = m; return -1; }
extern "C" const char *sdb_panoramic_last_error(void) { return g_perr.c_str(); }

namespace {
struct Nccl {
  void *h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  bool load()
  {
    if (h) return true;
    const char *names[] = { getenv("SDB_NCCL_LIB"), "libnccl.so.2", "libnccl.so" };
    for (const char *n : names) { if (n && (h = dlopen(n, RTLD_NOW | RTLD_GLOBAL))) break; }
    if (!h) return false;
#define SYM(f, s) f = (decltype(f)) dlsym(h, s)
    SYM(GetUniqueId, "ncclGetUniqueId"); SYM(CommInitRank, "ncclCommInitRank"); SYM(CommDestroy, "ncclCommDestroy");
    SYM(GroupStart, "ncclGroupStart"); SYM(GroupEnd, "ncclGroupEnd"); SYM(Send, "ncclSend"); SYM(Recv, "ncclRecv");
    SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
    return GetUniqueId && CommInitRank && CommDestroy && GroupStart && GroupEnd && Send && Recv;
  }
};
Nccl g_nccl;

void shard(size_t n_hops, int world, int rank, size_t *lo, size_t *hi)
{
  const size_t base = n_hops / (size_t) world, rem = n_hops % (size_t) world;
  *lo = (size_t) rank * base + std::min<size_t>((size_t) rank, rem);
  *hi = *lo + base + ((size_t) rank < rem ? 1 : 0);
}
}  // namespace

// One rank's outputs of a sweep, section by section (rows = hops of the shard):
//   j0[rows] i32 | nb[rows] i32 | va[rows][mb] f32 | vc[rows][mb] f32 | ccnt[rows] i32 | chan[rows][cap]   (last two: detector)
// Rank 0 owns the GLOBAL arrays ([n_hops] rows, hop order) and writes its own shard straight into rows [0, hi_0);
// the peers own arrays of their shard's size and send them section by section to the rows [lo_r, hi_r) of rank 0
// (one NCCL group of ncclSend / ncclRecv): nothing is unpacked or copied after the gather.
struct HopLists {
  DevBuf<int32_t> j0, nb; DevBuf<float> va, vc;
  DevBuf<int32_t> ccnt; DevBuf<sdb_detected_channel> chan;
};

// Rank 0, after the gather: the per-hop channel lists ([hops][cap], mostly empty) packed hop after hop, so that the
// read-back carries the channels that exist (a few hundred KB) instead of the 3.7 MB array they sit in.
//   k_chan_offsets: one CTA; off[h] = sum of the counts before hop h, off[n_hops] = total
//   k_chan_dense  : one block per hop copies its channels to dense[off[h] ...] while they fit in dense_cap
__global__ void k_chan_offsets(const int32_t *__restrict__ cnt, int n_hops, int32_t *__restrict__ off)
{
  __shared__ int s_w[32];
  __shared__ int s_carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n_hops; base += 1024) {
    const int h = base + tid;
    const int v = h < n_hops ? cnt[h] : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = s_w[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += t; }
      s_w[lane] = w;
    }
    __syncthreads();
    const int carry = s_carry;
    if (h < n_hops) off[h] = carry + (warp ? s_w[warp - 1] : 0) + incl - v;
    __syncthreads();
    if (tid == 0) s_carry = carry + s_w[31];
    __syncthreads();
  }
  if (tid == 0) off[n_hops] = s_carry;
}

__global__ void k_chan_dense(const int32_t *__restrict__ cnt, const int32_t *__restrict__ off,
                             const sdb_detected_channel *__restrict__ chan, int cap, sdb_detected_channel *__restrict__ dense,
                             int dense_cap)
{
  const int h = blockIdx.x, n = cnt[h], o = off[h];
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (o + i < dense_cap) dense[o + i] = chan[(size_t) h * cap + i];
}

struct sdb_panoramic {
  sdb_panoramic_params prm;
  int rank = 0, world = 1;
  ncclComm_t comm = nullptr;
  Stream stream;
  sdb_engine_t *eng = nullptr; size_t eng_hops = 0;
  sdb_sview_t *view = nullptr;
  size_t mb = 0;
  HopLists lists;
  DevBuf<double> d_centers;
  DevBuf<float> d_db;
  // rank 0, detector: the gathered channel lists land in pinned host memory behind ev_chan
  PinnedBuf<int32_t> h_off; PinnedBuf<sdb_detected_channel> h_chan; size_t n_hops_last = 0;
  DevBuf<int32_t> d_off; DevBuf<sdb_detected_channel> d_dense; size_t dense_cap = 0;
  std::vector<sdb_detected_channel> h_full; std::vector<int32_t> h_full_cnt; bool full_valid = false;   // overflow path
  std::vector<double> centers_last;            // hop centres of the last sweep (already on the device)
  Event ev_chan, ev_eng; bool chan_pending = false;   // chan_pending: ev_chan recorded, not yet synchronised
  Event ev[4];                                          // phase times of the last sweep
  sdb_panoramic_timing last{};
};

#define PCK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) return pfail(std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)
#define NCK(x) do { ncclResult_t r_ = (x); if (r_ != ncclSuccess) return pfail(std::string(#x) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "nccl error")); } while (0)

extern "C" int sdb_panoramic_unique_id(void *id128)
{
  if (!id128) return pfail("null id");
  if (!g_nccl.load()) return pfail("libnccl.so.2 not found (set SDB_NCCL_LIB)");
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  NCK(g_nccl.GetUniqueId(&id));
  memcpy(id128, &id, sizeof(id));
  return 0;
}

extern "C" sdb_panoramic_t *sdb_panoramic_new(const sdb_panoramic_params *p, int rank, int world, const void *id128)
{
  if (!p || world < 1 || rank < 0 || rank >= world) { g_perr = "invalid arguments"; return nullptr; }
  if (sdb_device_count() <= 0) { g_perr = "no CUDA device: sigdigger_b200 has no CPU fallback"; return nullptr; }
  if (!(p->freq_max > p->freq_min) || !(p->fft_bandwidth > 0) || p->psd_size < 16 || (p->psd_size & (p->psd_size - 1))) {
    g_perr = "invalid sweep parameters"; return nullptr;
  }
  if (cudaSetDevice(p->device) != cudaSuccess) { g_perr = "cudaSetDevice failed"; return nullptr; }
  sdb_panoramic *s = new sdb_panoramic();
  s->prm = *p; s->rank = rank; s->world = world;
  if (s->prm.channel_cap == 0) s->prm.channel_cap = 64;
  if (world > 1) {
    if (!id128 || !g_nccl.load()) { g_perr = "NCCL unavailable or no unique id"; delete s; return nullptr; }
    ncclUniqueId id; memcpy(&id, id128, sizeof(id));
    if (g_nccl.CommInitRank(&s->comm, world, id, rank) != ncclSuccess) { g_perr = "ncclCommInitRank failed"; delete s; return nullptr; }
  }
  bool ok = s->stream.create(cudaStreamNonBlocking) == cudaSuccess && s->ev_chan.create() == cudaSuccess &&
            s->ev_eng.create() == cudaSuccess;
  for (auto &e : s->ev) ok = ok && e.create(cudaEventDefault) == cudaSuccess;
  if (!ok) { g_perr = "CUDA stream or event creation failed"; sdb_panoramic_destroy(s); return nullptr; }
  s->view = sdb_sview_new(p->device);
  if (!s->view || sdb_sview_set_range(s->view, p->freq_min, p->freq_max, p->fft_bandwidth, p->rel_bw > 0 ? p->rel_bw : 0.5f)) {
    g_perr = "SpectrumView set-up failed"; sdb_panoramic_destroy(s); return nullptr;
  }
  s->mb = sdb_sview_max_bins(s->view);
  return s;
}

extern "C" void sdb_panoramic_destroy(sdb_panoramic_t *s)
{
  if (!s) return;
  cudaSetDevice(s->prm.device);
  if (s->stream) cudaStreamSynchronize(s->stream);
  if (s->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(s->comm);
  if (s->eng) sdb_engine_destroy(s->eng);
  if (s->view) sdb_sview_destroy(s->view);
  delete s;
}

static int ensure(sdb_panoramic *s, size_t n_hops, size_t n_local)
{
  const size_t rows = s->rank == 0 ? n_hops : n_local, mb = s->mb, cap = s->prm.channel_cap;
  // The row count of each group of buffers is the size of one of them, released first and allocated last: after a
  // failed allocation it is 0, so the next sweep allocates the whole group again.
  HopLists &l = s->lists;
  if (l.j0.size() < rows) {
    PCK(cudaStreamSynchronize(s->stream));
    l.j0.release();
    s->n_hops_last = 0;                    // the lists of the last sweep are gone
    PCK(l.nb.alloc(rows)); PCK(l.va.alloc(rows * mb)); PCK(l.vc.alloc(rows * mb));
    if (s->prm.detect) { PCK(l.ccnt.alloc(rows)); PCK(l.chan.alloc(rows * cap)); }
    PCK(l.j0.alloc(rows));
  }
  if (s->d_centers.size() < n_hops) {
    PCK(cudaStreamSynchronize(s->stream));
    PCK(s->d_centers.alloc(n_hops));
  }
  if (s->rank == 0 && s->prm.detect && s->h_off.size() < n_hops + 1) {
    PCK(cudaStreamSynchronize(s->stream));
    s->h_off.release();                    // sdb_panoramic_read_channels reads nothing until the lists are complete
    // room for 8 channels per hop on average (the lists hold up to `cap` each); a sweep that finds more is read
    // back in full, on demand (sdb_panoramic_read_channels)
    s->dense_cap = std::min(n_hops * cap, 8 * n_hops + 256);
    if (const char *env = getenv("SDB_PANORAMIC_DENSE_CAP")) {        // tests: force the overflow path
      const long v = atol(env);
      if (v >= 1) s->dense_cap = std::min(s->dense_cap, (size_t) v);
    }
    PCK(s->h_chan.alloc(s->dense_cap)); PCK(s->d_off.alloc(n_hops + 1)); PCK(s->d_dense.alloc(s->dense_cap));
    PCK(s->h_off.alloc(n_hops + 1));
  }
  if (n_local && (!s->eng || s->eng_hops != n_local)) {
    if (s->eng) sdb_engine_destroy(s->eng);
    sdb_engine_params ep; memset(&ep, 0, sizeof(ep));
    ep.n_streams = (uint32_t) n_local; ep.psd_size = s->prm.psd_size; ep.psd_window = s->prm.psd_window;
    ep.max_feed = s->prm.psd_size * (s->prm.frames_per_hop ? s->prm.frames_per_hop : 1); ep.device = s->prm.device;
    ep.flags = s->prm.detect ? 0 : SDB_FLAG_PSD_SHIFT_DB;       // the detector reads the linear PSD
    s->eng = sdb_engine_new(&ep, s->prm.fft_bandwidth);
    if (!s->eng) return pfail(sdb_last_error());
    if (s->prm.detect &&
        sdb_engine_set_channel_detector(s->eng, s->prm.det_alpha, 0.0f, s->prm.det_gamma, s->prm.det_snr,
                                        s->prm.det_min_bins ? s->prm.det_min_bins : 2))
      return pfail(sdb_last_error());
    if (sdb_engine_commit(s->eng)) return pfail(sdb_last_error());
    s->eng_hops = n_local;
  }
  return 0;
}

// hops_local: this rank's contiguous shard [hi - lo][psd_size] (device pointer if on_device), one window per hop.
// Everything between the first and the last event is queued on streams: the engine's feed (its own streams), then
// on s->stream behind an event the dB pass, the projection, the channel-list conversion, the NCCL group and rank 0's
// accumulate + fill.  The host blocks once, at the end, for the phase times.
static int sweep_impl(sdb_panoramic *s, const sdb_complex *hops_local, int on_device, const double *centers_all,
                      size_t n_hops)
{
  if (!s || !centers_all || n_hops == 0) return pfail("invalid arguments");
  PCK(cudaSetDevice(s->prm.device));
  size_t lo, hi;
  shard(n_hops, s->world, s->rank, &lo, &hi);
  const size_t n_local = hi - lo, N = s->prm.psd_size, mb = s->mb, cap = s->prm.channel_cap;
  if (n_local && !hops_local) return pfail("null hop buffer");
  if (ensure(s, n_hops, n_local)) return -1;
  cudaStream_t st = s->stream;
  HopLists &l = s->lists;
  const size_t row0 = s->rank == 0 ? lo : 0;          // rank 0 writes into the global arrays (lo = 0 there)
  PCK(cudaEventRecord(s->ev[0], st));
  if (s->centers_last.size() != n_hops || memcmp(s->centers_last.data(), centers_all, n_hops * sizeof(double))) {
    s->centers_last.assign(centers_all, centers_all + n_hops);       // a scanner repeats its hop plan sweep after sweep
    PCK(cudaMemcpyAsync(s->d_centers, s->centers_last.data(), n_hops * sizeof(double), cudaMemcpyHostToDevice, st));
  }
  if (n_local) {
    // frames_per_hop > 1: the detector averages over the hop's frames, the view takes the last one
    const size_t F = s->prm.frames_per_hop ? s->prm.frames_per_hop : 1, L = N * F;
    if (on_device ? sdb_engine_feed_device(s->eng, hops_local, L, L) : sdb_engine_feed_host(s->eng, hops_local, L, L))
      return pfail(sdb_last_error());
    if (sdb_engine_join(s->eng)) return pfail(sdb_last_error());
    PCK(cudaEventRecord(s->ev_eng, (cudaStream_t) sdb_engine_stream(s->eng)));
    PCK(cudaStreamWaitEvent(st, s->ev_eng, 0));
    // the view takes the hop's last frame; with the detector on, the engine keeps the linear PSD and the projection
    // converts what it reads (fftshift + dB, Suscan/Messages/PSDMessage.cpp:32-38)
    const float *psd = sdb_engine_psd_device(s->eng) + (F - 1) * N;
    int rc = sdb_sview_project_async(s->view, st, psd, N, L, s->prm.detect ? 1 : 0, s->d_centers + lo, n_local, 1,
                                     l.j0 + row0, l.nb + row0, l.va + row0 * mb, l.vc + row0 * mb);
    if (rc == 1) {
      // geometry outside the tiled kernel (a hop narrower than two view bins, or very wide): dB frames, contiguous
      if (s->d_db.size() < n_local * N) {
        PCK(cudaStreamSynchronize(st));
        PCK(s->d_db.alloc(n_local * N));
      }
      if (s->prm.detect) {
        for (size_t h = 0; h < (F == 1 ? 1 : n_local); ++h)
          if (sdb_psd_shift_db_async(st, psd + h * L, s->d_db + h * N, F == 1 ? n_local : 1, (uint32_t) N))
            return pfail(sdb_last_error());
      } else {
        PCK(cudaMemcpy2DAsync(s->d_db, N * sizeof(float), psd, L * sizeof(float), N * sizeof(float), n_local,
                              cudaMemcpyDeviceToDevice, st));
      }
      rc = sdb_sview_project_async(s->view, st, s->d_db, N, N, 0, s->d_centers + lo, n_local, 1, l.j0 + row0,
                                   l.nb + row0, l.va + row0 * mb, l.vc + row0 * mb);
    }
    if (rc) return pfail(rc == 1 ? "projection geometry not supported" : sdb_last_error());
    if (s->prm.detect &&
        sdb_engine_pack_channels_device(s->eng, s->d_centers + lo, l.chan + row0 * cap, cap, l.ccnt + row0, st))
      return pfail(sdb_last_error());
  }
  PCK(cudaEventRecord(s->ev[1], st));
  // ---- the one exchange of the path: every peer's sections go to their rows of rank 0's global arrays
  uint64_t gathered = 0;
  if (s->world > 1) {
    NCK(g_nccl.GroupStart());
    for (int r = 1; r < s->world; ++r) {
      if (s->rank != 0 && s->rank != r) continue;
      size_t rlo, rhi;
      shard(n_hops, s->world, r, &rlo, &rhi);
      const size_t cnt = rhi - rlo, at = s->rank == 0 ? rlo : 0;
      if (!cnt) continue;
      struct { void *p; size_t bytes; } sec[6] = {
        { l.j0 + at, cnt * sizeof(int32_t) }, { l.nb + at, cnt * sizeof(int32_t) },
        { l.va + at * mb, cnt * mb * sizeof(float) }, { l.vc + at * mb, cnt * mb * sizeof(float) },
        { s->prm.detect ? (void *) (l.ccnt + at) : nullptr, cnt * sizeof(int32_t) },
        { s->prm.detect ? (void *) (l.chan + at * cap) : nullptr, cnt * cap * sizeof(sdb_detected_channel) } };
      for (auto &q : sec) {
        if (!q.p) continue;
        if (s->rank == 0) { NCK(g_nccl.Recv(q.p, q.bytes, ncclUint8, r, s->comm, st)); gathered += q.bytes; }
        else NCK(g_nccl.Send(q.p, q.bytes, ncclUint8, 0, s->comm, st));
      }
    }
    NCK(g_nccl.GroupEnd());
  }
  PCK(cudaEventRecord(s->ev[2], st));
  s->last.gather_bytes = gathered;
  if (s->rank == 0) {
    // rows are in global hop order already: accumulate + fill exactly as one sequential feed() series
    if (sdb_sview_accumulate_async(s->view, st, l.j0, l.nb, l.va, l.vc, n_hops)) return pfail(sdb_last_error());
    if (s->prm.detect) {
      k_chan_offsets<<<1, 1024, 0, st>>>(l.ccnt, (int) n_hops, s->d_off);
      k_chan_dense<<<(unsigned) n_hops, 64, 0, st>>>(l.ccnt, s->d_off, l.chan, (int) cap, s->d_dense, (int) s->dense_cap);
      PCK(cudaGetLastError());
      PCK(cudaMemcpyAsync(s->h_off, s->d_off, (n_hops + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      PCK(cudaMemcpyAsync(s->h_chan, s->d_dense, s->dense_cap * sizeof(sdb_detected_channel), cudaMemcpyDeviceToHost, st));
      PCK(cudaEventRecord(s->ev_chan, st));
      s->chan_pending = true; s->full_valid = false;
    }
    s->n_hops_last = n_hops;
  }
  PCK(cudaEventRecord(s->ev[3], st));
  PCK(cudaEventSynchronize(s->ev[3]));
  s->chan_pending = false;
  if (n_local && sdb_engine_sync(s->eng)) return pfail(sdb_last_error());
  float a = 0, b = 0, c = 0;
  cudaEventElapsedTime(&a, s->ev[0], s->ev[1]); cudaEventElapsedTime(&b, s->ev[1], s->ev[2]); cudaEventElapsedTime(&c, s->ev[2], s->ev[3]);
  s->last.psd_project_ms = a; s->last.gather_ms = b; s->last.accumulate_ms = c;
  s->last.n_hops_local = n_local;
  return 0;
}

extern "C" int sdb_panoramic_sweep_device(sdb_panoramic_t *s, const sdb_complex *hops_local_dev, const double *centers_all,
                                          size_t n_hops)
{ return sweep_impl(s, hops_local_dev, 1, centers_all, n_hops); }
extern "C" int sdb_panoramic_sweep_host(sdb_panoramic_t *s, const sdb_complex *hops_local, const double *centers_all,
                                        size_t n_hops)
{ return sweep_impl(s, hops_local, 0, centers_all, n_hops); }

extern "C" int sdb_panoramic_reset(sdb_panoramic_t *s)
{
  if (!s) return pfail("null");
  if (cudaSetDevice(s->prm.device) != cudaSuccess) return pfail("cudaSetDevice failed");
  return sdb_sview_reset_async(s->view, s->stream) ? pfail(sdb_last_error()) : 0;
}
extern "C" int sdb_panoramic_read(sdb_panoramic_t *s, float *psd, float *accum, float *count, size_t cap)
{
  if (!s) return pfail("null");
  if (s->rank != 0) return pfail("the stitched view lives on rank 0");
  return sdb_sview_read(s->view, psd, accum, count, cap) ? pfail(sdb_last_error()) : 0;
}
extern "C" uint32_t sdb_panoramic_size(const sdb_panoramic_t *s) { return s ? sdb_sview_size(s->view) : 0; }
extern "C" long sdb_panoramic_read_channels(sdb_panoramic_t *s, size_t hop, sdb_detected_channel *out, size_t cap)
{
  if (!s || s->rank != 0 || !s->prm.detect || hop >= s->n_hops_last || !s->h_off.size()) return -1;
  if (s->chan_pending) { cudaEventSynchronize(s->ev_chan); s->chan_pending = false; }
  const size_t n_hops = s->n_hops_last, pc = s->prm.channel_cap;
  if ((size_t) s->h_off[n_hops] <= s->dense_cap) {
    const size_t n = std::min(cap, (size_t) (s->h_off[hop + 1] - s->h_off[hop]));
    if (n && out) memcpy(out, s->h_chan + s->h_off[hop], n * sizeof(sdb_detected_channel));
    return (long) n;
  }
  // more channels than the packed read-back holds: fetch the whole [hops][cap] array once
  if (!s->full_valid) {
    if (cudaSetDevice(s->prm.device) != cudaSuccess) return -1;
    s->h_full.resize(n_hops * pc); s->h_full_cnt.resize(n_hops);
    if (cudaMemcpy(s->h_full_cnt.data(), s->lists.ccnt, n_hops * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(s->h_full.data(), s->lists.chan, n_hops * pc * sizeof(sdb_detected_channel), cudaMemcpyDeviceToHost) != cudaSuccess)
      return -1;
    s->full_valid = true;
  }
  const size_t n = std::min(cap, (size_t) s->h_full_cnt[hop]);
  if (n && out) memcpy(out, s->h_full.data() + hop * pc, n * sizeof(sdb_detected_channel));
  return (long) n;
}
extern "C" int sdb_panoramic_last_timing(const sdb_panoramic_t *s, sdb_panoramic_timing *t)
{
  if (!s || !t) return -1;
  *t = s->last;
  return 0;
}
extern "C" void sdb_panoramic_shard(size_t n_hops, int world, int rank, size_t *lo, size_t *hi) { shard(n_hops, world, rank, lo, hi); }
