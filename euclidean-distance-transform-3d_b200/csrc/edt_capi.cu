// edt_capi.cu -- host side of the C ABI declared in include/edt_b200.h.
//
// Plays the role of the reference's volume drivers (pyedt::_edt3dsq / _edt2dsq,
// src/edt.hpp:411-484, 632-678): it owns the pass order X -> Y -> Z over one float32
// volume that is transformed in place, but the "thread pool" is the CUDA grid and the
// passes are stream-ordered kernel launches.  No CPU fallback exists in this file.
#include "edt_host.h"
#include "edt_voxel_graph.cuh"
#include "edt_each.cuh"
#include "edt_slab.cuh"

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <dlfcn.h>
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

namespace edtb200 {
namespace host {

thread_local char g_error[512] = "";
thread_local LaterLaunch g_last_later;

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
  return code;
}

EncodeTiledFn tensor_map_encoder() {
  static std::once_flag once;
  static EncodeTiledFn encode = nullptr;
  std::call_once(once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      encode = reinterpret_cast<EncodeTiledFn>(fn);
    else
      cudaGetLastError();
  });
  return encode;
}

// ---- PassArith: the arithmetic of a later-axis pass, from a transform or from its samples ----

// Lowest set bit of v > 0 (a power of two); 0 for v <= 0 or not finite.
static double lowest_bit(double v) {
  if (!(v > 0.0) || !std::isfinite(v)) return 0.0;
  int e = 0;
  const double m = frexp(v, &e);                                   // v = m 2^e, m in [0.5, 1)
  const unsigned long long mant = (unsigned long long)ldexp(m, 53);
  return ldexp(1.0, e - 53 + __builtin_ctzll(mant));
}

// The rule both producers end in, for a pass with squared weight w2 over lines of n finite
// samples that are at most `top`, whole multiples of `unit` (as w2 is), and integers not above
// int_bound (-1: not known to be integers).
static PassArith pass_arith(double int_bound, double top, double unit, float w2, int64_t n) {
  const double reach = (double)w2 * (double)n * (double)n;
  PassArith a;
  a.int_hull = int_bound >= 0.0 && w2 == floorf(w2) && w2 >= 1.0f && w2 < 1048576.0f &&
               int_bound + reach < 2147483000.0;
  // w2 d^2 is exact in double (24 + 24 bits), so a sum is exact when it spans at most 53 bits from
  // `unit` up; then one fused multiply-add rounds what the reference rounds once (src/edt.hpp:232).
  a.exact = top + reach < 0x1p53 * unit;
  return a;
}

// The samples are what the passes along axes 0..k-1 made, at most the sum of w2 * n^2 over those
// axes (the factor 2 covers their float32 rounding); integers when every squared weight is one
// and the X pass's distances j * w[0] are integers below 2^24.  The unit:
//  - when the X pass is exact (every distance j * w[0] below 2^24 units of b0 = lowest_bit(w[0])),
//    its squares are multiples of b0^2, every w2 = fl32(w * w) is a multiple of its lowest set bit,
//    and float32 rounding keeps a multiple of a power of two P a multiple of P: so every sample and
//    candidate is a multiple of the least of b0^2 and those bits (1 or more for integer weights,
//    1/4 for weights of 0.5, ...);
//  - otherwise every positive sample is at least the least squared weight (the X pass's smallest
//    distance is one step), so half the float32 spacing there divides them all.
PassArith transform_arith(const float* w, const int64_t* n, int k) {
  double top = 0.0;
  float least = INFINITY;
  const double b0 = lowest_bit((double)w[0]);
  double unit = b0 * b0;
  const bool x_exact = b0 > 0.0 && (double)w[0] * (double)n[0] < 16777216.0 * b0;
  bool integral = (double)w[0] == floor((double)w[0]) && (double)w[0] * (double)n[0] < 16777216.0;
  for (int i = 0; i <= k; ++i) {
    const float w2 = w[i] * w[i];
    if (i < k) {
      top += (double)w2 * (double)n[i] * (double)n[i];
      integral = integral && w2 == floorf(w2) && w2 >= 1.0f;
    }
    least = fminf(least, w2);
    if (i > 0) unit = fmin(unit, lowest_bit((double)w2));
  }
  if (!x_exact || !(unit > 0.0)) unit = 0.5 * ((double)nextafterf(least, INFINITY) - (double)least);
  return pass_arith(integral ? top : -1.0, 2.0 * top, unit, w[k] * w[k], n[k]);
}

// Every sample and every w2 d^2 is a multiple of the least of 2^low and w2's lowest set bit; the
// samples are integers when low >= 0.
PassArith sampled_arith(float fmax, int low, float w, int64_t n) {
  const float w2 = w * w;
  double unit = lowest_bit((double)w2);
  if (low < 1024) unit = fmin(unit, ldexp(1.0, low));
  return pass_arith(low >= 0 ? (double)fmax : -1.0, fmax, unit, w2, n);
}

cudaError_t scratch_alloc(DeviceCache& dc, void** p, size_t bytes, cudaStream_t stream) {
  if (dc.pool) return cudaMallocFromPoolAsync(p, bytes, dc.pool, stream);
  return cudaMallocAsync(p, bytes, stream);
}

// Device table T[0..count) for weight w, cached per device.  Built once on `stream`; other
// streams wait on the build event, so no host synchronisation and no per-call allocation.
// When all slots are taken the least recently used table is retired: the retiring stream waits
// for the last kernel of every stream that used the table (one event per user stream) and the
// buffer is freed in stream order -- no device-wide synchronisation.  The table returned stays
// pinned until step_table_used: another thread's launch that needs a new table must not retire it
// while the kernel that reads it is not queued yet (its use is not recorded), so pinned tables are
// never victims -- when every slot is pinned, the caller waits for one to be released.
int step_table(DeviceCache& dc, float w, int count, cudaStream_t stream, const float** out) {
  std::unique_lock<std::mutex> guard(dc.lock);
  uint32_t wbits;
  memcpy(&wbits, &w, sizeof(wbits));
  DeviceCache::Table* hit = nullptr;
  DeviceCache::Table* victim = nullptr;
  for (;;) {
    for (auto& t : dc.tables) {
      if (t.data && t.wbits == wbits && t.count >= count) { hit = &t; break; }
      if (!t.pinned && (!victim || t.stamp < victim->stamp)) victim = &t;
    }
    if (hit || victim) break;
    dc.table_unpinned.wait(guard);
  }
  if (!hit) {
    DeviceCache::Table& t = *victim;
    if (t.data) {
      if (t.many_users) CUDA_TRY(cudaDeviceSynchronize());    // more user streams than tracked: rare
      for (int u = 0; u < DeviceCache::Table::kUsers; ++u)
        if (t.user_set[u]) CUDA_TRY(cudaStreamWaitEvent(stream, t.used[u], 0));
      if (t.ready) CUDA_TRY(cudaStreamWaitEvent(stream, t.ready, 0));
      CUDA_TRY(cudaFreeAsync(t.data, stream));
      t.data = nullptr;
      for (int u = 0; u < DeviceCache::Table::kUsers; ++u) t.user_set[u] = false;
      t.many_users = false;
    }
    const int cap = count < 4096 ? 4096 : count;
    CUDA_TRY(scratch_alloc(dc, reinterpret_cast<void**>(&t.data), sizeof(float) * (size_t)cap, stream));
    if (!t.ready) CUDA_TRY(cudaEventCreateWithFlags(&t.ready, cudaEventDisableTiming));
    step_table_kernel<<<1, 32, 0, stream>>>(w, cap, t.data);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(t.ready, stream));
    t.count = cap; t.wbits = wbits; t.built_on = stream;
    hit = &t;
  } else if (hit->built_on != stream) {
    CUDA_TRY(cudaStreamWaitEvent(stream, hit->ready, 0));
  }
  hit->stamp = ++dc.table_clock;
  ++hit->pinned;
  *out = hit->data;
  return 0;
}

// Called once the kernel that reads table `data` has been queued on `stream` (queued), or when its
// launch failed (nothing to record).  A pinned table is never retired, so `data` still names it.
int step_table_used(DeviceCache& dc, const float* data, cudaStream_t stream, bool queued) {
  std::lock_guard<std::mutex> guard(dc.lock);
  for (auto& t : dc.tables) {
    if (t.data != data) continue;
    if (--t.pinned == 0) dc.table_unpinned.notify_all();
    if (!queued) return 0;
    int slot = -1;
    for (int u = 0; u < DeviceCache::Table::kUsers; ++u)
      if (t.user_set[u] && t.user[u] == stream) { slot = u; break; }
    if (slot < 0)
      for (int u = 0; u < DeviceCache::Table::kUsers; ++u)
        if (!t.user_set[u]) { slot = u; break; }
    if (slot < 0) { t.many_users = true; return 0; }
    if (!t.used[slot]) CUDA_TRY(cudaEventCreateWithFlags(&t.used[slot], cudaEventDisableTiming));
    CUDA_TRY(cudaEventRecord(t.used[slot], stream));
    t.user[slot] = stream; t.user_set[slot] = true;
    return 0;
  }
  return 0;
}

// The last CTA of an X launch is the one that draws ticket gridDim.x - 1, and it resets the counter
// and the ticket: two launches that shared them at the same time (device-resident calls on two
// streams take no lock) would leave the ticket off by the other grid's CTAs for good, and grids
// smaller than that offset would never publish again.  So every launch takes the next pair of a
// ring; a pair comes round again only after kStatSlots more launches, and its previous launch has
// left it at zero by then unless that many X passes run at once.
RunStat run_stat(DeviceCache& dc, unsigned long long voxels) {
  RunStat st;
  memset(&st, 0, sizeof(st));
  std::lock_guard<std::mutex> guard(dc.lock);
  if (!dc.stat_slots) return st;
  char* slot = static_cast<char*>(dc.stat_slots) + 16 * (size_t)(dc.stat_next++ % DeviceCache::kStatSlots);
  st.counter = reinterpret_cast<unsigned long long*>(slot);
  st.ticket = reinterpret_cast<unsigned int*>(slot + 8);
  st.publish = dc.stat_publish_dev;
  st.voxels = voxels;
  return st;
}

}  // namespace host
}  // namespace edtb200

namespace {

using namespace edtb200::host;

constexpr int kMaxDevices = 64;
DeviceCache g_cache[kMaxDevices];

// ---- host <-> device staging for pageable host memory --------------------------------
// numpy arrays are pageable: a plain cudaMemcpy of 512 MiB then runs at a fraction of the PCIe
// rate (the driver stages it through small internal buffers, and a freshly allocated output
// array is also page-faulted in by that single thread).  Pinned callers are copied directly;
// pageable ones go through three 32 MiB pinned buffers that a few host threads fill / drain in
// parallel while the DMA engine moves the previous chunk.
class CopyPool {
 public:
  explicit CopyPool(int n) : n_(n) {
    for (int i = 0; i < n_; ++i) threads_.emplace_back([this, i] { loop(i); });
  }
  ~CopyPool() {
    { std::lock_guard<std::mutex> l(m_); stop_ = true; ++epoch_; }
    cv_.notify_all();
    for (auto& t : threads_) t.join();
  }
  int size() const { return n_; }
  // run fn(i) for i in [0, n) on the pool and wait
  void run(const std::function<void(int)>& fn) {
    std::unique_lock<std::mutex> l(m_);
    fn_ = &fn; pending_ = n_; ++epoch_;
    cv_.notify_all();
    done_.wait(l, [this] { return pending_ == 0; });
    fn_ = nullptr;
  }
 private:
  void loop(int i) {
    unsigned long seen = 0;
    for (;;) {
      const std::function<void(int)>* fn;
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return epoch_ != seen; });
        seen = epoch_;
        if (stop_) return;
        fn = fn_;
      }
      (*fn)(i);
      {
        std::lock_guard<std::mutex> l(m_);
        if (--pending_ == 0) done_.notify_all();
      }
    }
  }
  int n_;
  std::vector<std::thread> threads_;
  std::mutex m_;
  std::condition_variable cv_, done_;
  const std::function<void(int)>* fn_ = nullptr;
  int pending_ = 0;
  unsigned long epoch_ = 0;
  bool stop_ = false;
};

// Per device, two pools and two sets of staging buffers: [0] for copies towards the device, [1]
// for copies back, so that a batch (edtb200_transform_batch) can drive both directions at once
// from two host threads, and calls on different devices never share a pool.  Created on first use
// (under g_init); used only by the holder of the device's host_call lock and its batch helper.
std::mutex g_init;
CopyPool* g_pools[2][kMaxDevices] = {};

// A box of host rows: `rows` rows of `width` bytes, row r at host + r * pitch.  Its device copy is
// packed (row r at r * width), so byte i of the box is device byte i.  A contiguous buffer is the
// box of one row.
struct HostBox {
  char* host;
  size_t width, pitch, rows;
  size_t bytes() const { return width * rows; }
  bool packed() const { return rows == 1 || pitch == width; }
};

// Copies box bytes [off, off + n) between the box's host rows and `packed`, which holds box byte off
// at its start; to_host: packed -> host rows.
void copy_box_bytes(char* packed, const HostBox& b, size_t off, size_t n, bool to_host) {
  while (n) {
    const size_t r = off / b.width, c = off % b.width, len = b.width - c < n ? b.width - c : n;
    char* h = b.host + r * b.pitch + c;
    if (to_host) memcpy(h, packed, len);
    else memcpy(packed, h, len);
    packed += len; off += len; n -= len;
  }
}

// Box bytes [off, off + bytes) between the host rows and the staging buffer `stage`, split over
// the device's copy pool for direction dir (0: towards the device, gathering; 1: back, scattering).
void parallel_copy(char* stage, const HostBox& b, size_t off, size_t bytes, int dir, int device) {
  CopyPool*& g_pool = g_pools[dir][device];
  if (!g_pool) {
    std::lock_guard<std::mutex> guard(g_init);
    unsigned hw = std::thread::hardware_concurrency();
    // a memcpy of pageable memory is bound by one core's page walks, so the copy is split over host
    // threads; beyond a couple of dozen threads memory bandwidth, not cores, limits it (the count is
    // not tuned per host: EDTB200_COPY_THREADS overrides it, tools/pageable_e2e.py times it)
    int n = hw >= 48 ? 24 : (hw >= 32 ? 16 : (hw >= 16 ? 8 : (hw >= 4 ? 4 : 1)));
    if (const char* e = getenv("EDTB200_COPY_THREADS")) n = std::max(1, std::min(64, atoi(e)));
    g_pool = new CopyPool(n);
  }
  const int n = g_pool->size();
  const size_t slice = ((bytes + n - 1) / n + 4095) & ~size_t(4095);
  g_pool->run([&](int i) {
    const size_t s = slice * (size_t)i;
    if (s < bytes) copy_box_bytes(stage + s, b, off + s, bytes - s < slice ? bytes - s : slice, dir == 1);
  });
}

// size of one staging buffer (EDTB200_STAGE_MB, 4..256, default 32) and how many rotate
const size_t kStageBytes = [] {
  size_t mb = 32;
  if (const char* e = getenv("EDTB200_STAGE_MB")) mb = (size_t)std::max(4, std::min(256, atoi(e)));
  return mb << 20;
}();
constexpr int kStages = 3;
struct StageBuffers {
  void* buf[kStages] = {nullptr, nullptr, nullptr};
  cudaEvent_t ev[kStages] = {nullptr, nullptr, nullptr};
};
StageBuffers g_stage[2][kMaxDevices];

bool host_pointer_is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}

int ensure_stage(int device, int dir) {
  StageBuffers& sb = g_stage[dir][device];
  for (int i = 0; i < kStages; ++i) {
    if (!sb.buf[i]) CUDA_TRY(cudaHostAlloc(&sb.buf[i], kStageBytes, cudaHostAllocDefault));
    if (!sb.ev[i]) CUDA_TRY(cudaEventCreateWithFlags(&sb.ev[i], cudaEventDisableTiming));
  }
  return 0;
}

// The box copied directly by the DMA engine: one copy when it is packed, else one 2-D copy, or one
// copy per row where a row pitch exceeds what cudaMemcpy2DAsync takes.
int copy_box_direct(char* dev, const HostBox& b, int device, cudaStream_t stream, bool to_host) {
  const cudaMemcpyKind kind = to_host ? cudaMemcpyDeviceToHost : cudaMemcpyHostToDevice;
  if (b.packed()) {
    CUDA_TRY(to_host ? cudaMemcpyAsync(b.host, dev, b.bytes(), kind, stream)
                     : cudaMemcpyAsync(dev, b.host, b.bytes(), kind, stream));
    return 0;
  }
  int max_pitch = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&max_pitch, cudaDevAttrMaxPitch, device));
  if (b.pitch <= (size_t)max_pitch) {
    CUDA_TRY(to_host ? cudaMemcpy2DAsync(b.host, b.pitch, dev, b.width, b.width, b.rows, kind, stream)
                     : cudaMemcpy2DAsync(dev, b.width, b.host, b.pitch, b.width, b.rows, kind, stream));
    return 0;
  }
  for (size_t r = 0; r < b.rows; ++r) {
    char* h = b.host + r * b.pitch;
    char* d = dev + r * b.width;
    CUDA_TRY(to_host ? cudaMemcpyAsync(h, d, b.width, kind, stream) : cudaMemcpyAsync(d, h, b.width, kind, stream));
  }
  return 0;
}

// host box (pageable or pinned) -> packed device buffer, stream-ordered; returns after the last
// chunk is queued.  Pageable rows are gathered into the staging buffers, a row longer than one
// buffer in several pieces.
int upload_box(void* dst_dev, const HostBox& box, int device, cudaStream_t stream) {
  const size_t bytes = box.bytes();
  char* dst = static_cast<char*>(dst_dev);
  if (bytes < (size_t(4) << 20) || host_pointer_is_pinned(box.host)) return copy_box_direct(dst, box, device, stream, false);
  int rc = ensure_stage(device, 0);
  if (rc) return rc;
  StageBuffers& sb = g_stage[0][device];
  size_t off = 0;
  for (int k = 0; off < bytes; ++k) {
    const int b = k % kStages;
    const size_t n = bytes - off < kStageBytes ? bytes - off : kStageBytes;
    // the DMA out of this buffer must have finished -- also the one queued by an EARLIER upload:
    // inside a batch the previous volume's copies may still be waiting in the stream
    CUDA_TRY(cudaEventSynchronize(sb.ev[b]));
    parallel_copy(static_cast<char*>(sb.buf[b]), box, off, n, 0, device);
    CUDA_TRY(cudaMemcpyAsync(dst + off, sb.buf[b], n, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaEventRecord(sb.ev[b], stream));
    off += n;
  }
  return 0;
}

// packed device buffer -> host box (pageable or pinned); complete on return for the pageable case
int download_box(const HostBox& box, const void* src_dev, int device, cudaStream_t stream) {
  const size_t bytes = box.bytes();
  const char* src = static_cast<const char*>(src_dev);
  if (bytes < (size_t(4) << 20) || host_pointer_is_pinned(box.host))
    return copy_box_direct(const_cast<char*>(src), box, device, stream, true);
  int rc = ensure_stage(device, 1);
  if (rc) return rc;
  StageBuffers& sb = g_stage[1][device];
  size_t off = 0, prev_off = 0, prev_n = 0;
  int prev_b = -1;
  for (int k = 0; off < bytes || prev_b >= 0; ++k) {
    int b = -1;
    size_t n = 0;
    if (off < bytes) {
      b = k % kStages;
      n = bytes - off < kStageBytes ? bytes - off : kStageBytes;
      CUDA_TRY(cudaMemcpyAsync(sb.buf[b], src + off, n, cudaMemcpyDeviceToHost, stream));
      CUDA_TRY(cudaEventRecord(sb.ev[b], stream));
    }
    if (prev_b >= 0) {                                             // drain the chunk queued one step earlier
      CUDA_TRY(cudaEventSynchronize(sb.ev[prev_b]));
      parallel_copy(static_cast<char*>(sb.buf[prev_b]), box, prev_off, prev_n, 1, device);
    }
    prev_b = b; prev_off = off; prev_n = n;
    off += n;
  }
  return 0;
}

// contiguous host buffers: the box of one row
int upload(void* dst_dev, const void* src_host, size_t bytes, int device, cudaStream_t stream) {
  return upload_box(dst_dev, HostBox{static_cast<char*>(const_cast<void*>(src_host)), bytes, bytes, 1}, device, stream);
}

int download(void* dst_host, const void* src_dev, size_t bytes, int device, cudaStream_t stream) {
  return download_box(HostBox{static_cast<char*>(dst_host), bytes, bytes, 1}, src_dev, device, stream);
}

// The device's private non-blocking stream, created on first use by the holder of host_call.
cudaError_t private_stream(DeviceCache& dc) {
  return dc.stream ? cudaSuccess : cudaStreamCreateWithFlags(&dc.stream, cudaStreamNonBlocking);
}

// Restores the calling thread's current CUDA device when an entry point returns (callers such as
// PyTorch rely on "their" current device staying put).
struct DeviceGuard {
  int saved = -1;
  DeviceGuard() { if (cudaGetDevice(&saved) != cudaSuccess) { cudaGetLastError(); saved = -1; } }
  ~DeviceGuard() { if (saved >= 0) cudaSetDevice(saved); }
};

int probe(int device, DeviceCache** out) {
  if (device < 0 || device >= kMaxDevices) return fail(EDTB200_EINVAL, "bad device %d", device);
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    return fail(EDTB200_ECUDA, "no usable CUDA device (%s); this library has no CPU fallback",
                e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
  if (device >= count) return fail(EDTB200_EINVAL, "device %d out of range (%d visible)", device, count);
  DeviceCache& dc = g_cache[device];
  CUDA_TRY(cudaSetDevice(device));
  std::lock_guard<std::mutex> guard(dc.lock);
  if (!dc.probed) {
    CUDA_TRY(cudaDeviceGetAttribute(&dc.sm_count, cudaDevAttrMultiProcessorCount, device));
    CUDA_TRY(cudaDeviceGetAttribute(&dc.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    // Stream-ordered scratch (voxel-graph grids, long-line temporaries, step tables) comes from a
    // PRIVATE pool: the process-wide default pool -- which the host application (PyTorch, CuPy)
    // may share -- keeps its own settings.  The pool keeps up to EDTB200_POOL_KEEP_MB (default
    // 1024) between calls so that repeated transforms do not go back to the driver;
    // edtb200_release() trims it to nothing.
    cudaMemPoolProps props;
    memset(&props, 0, sizeof(props));
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = device;
    if (cudaMemPoolCreate(&dc.pool, &props) == cudaSuccess) {
      unsigned long long keep = 1024ull << 20;
      if (const char* env = getenv("EDTB200_POOL_KEEP_MB")) keep = strtoull(env, nullptr, 10) << 20;
      cudaMemPoolSetAttribute(dc.pool, cudaMemPoolAttrReleaseThreshold, &keep);
    } else {
      dc.pool = nullptr;                 // fall back to the default pool, settings untouched
    }
    cudaGetLastError();
    // run statistic of the first-axis pass: a ring of device counter / ticket pairs and two mapped
    // host words
    void* stat = nullptr;
    void* host = nullptr;
    const size_t stat_bytes = 16 * (size_t)DeviceCache::kStatSlots;
    if (cudaMalloc(&stat, stat_bytes) == cudaSuccess && cudaMemset(stat, 0, stat_bytes) == cudaSuccess &&
        cudaHostAlloc(&host, 64, cudaHostAllocMapped | cudaHostAllocPortable) == cudaSuccess) {
      memset(host, 0, 64);
      void* host_dev = nullptr;
      if (cudaHostGetDevicePointer(&host_dev, host, 0) == cudaSuccess) {
        dc.stat_slots = stat;
        dc.stat_publish_host = static_cast<volatile unsigned long long*>(host);
        dc.stat_publish_dev = static_cast<unsigned long long*>(host_dev);
      }
    }
    cudaGetLastError();
    dc.probed = true;
  }
  *out = &dc;
  return 0;
}

int check_dims(int label_bytes, int ndim, int64_t& sx, int64_t& sy, int64_t& sz) {
  if (!(label_bytes == 1 || label_bytes == 2 || label_bytes == 4 || label_bytes == 8))
    return fail(EDTB200_EINVAL, "label_bytes must be 1, 2, 4 or 8 (got %d)", label_bytes);
  if (ndim < 1 || ndim > 3) return fail(EDTB200_EINVAL, "ndim must be 1, 2 or 3 (got %d)", ndim);
  if (ndim < 3) sz = 1;
  if (ndim < 2) sy = 1;
  if (sx < 0 || sy < 0 || sz < 0) return fail(EDTB200_EINVAL, "negative size");
  const int64_t lim = (int64_t)1 << 30;
  if (sx > lim || sy > lim || sz > lim) return fail(EDTB200_ELIMIT, "axis longer than 2^30");
  return 0;
}

int check_weights(int ndim, const float w[3]) {
  for (int k = 0; k < ndim; ++k)
    if (!(std::isfinite(w[k]) && w[k] > 0.0f))
      return fail(EDTB200_EINVAL, "the weight of axis %d must be finite and > 0 (got %g)", k, (double)w[k]);
  return 0;
}

// A stack of `count` volumes of `vol` voxels, `per_voxel` values each, holds at most 2^62 values.
int check_stack(int64_t vol, int64_t count, int64_t per_voxel) {
  if (vol > 0 && count > ((int64_t)1 << 62) / (vol * per_voxel))
    return fail(EDTB200_ELIMIT, "too many voxels in the stack");
  return 0;
}

int check_float_labels(int flags, int label_bytes) {
  if ((flags & EDTB200_LABELS_FLOAT) && label_bytes != 4 && label_bytes != 8)
    return fail(EDTB200_EINVAL, "EDTB200_LABELS_FLOAT needs 4- or 8-byte labels");
  return 0;
}

bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
  return (const char*)a < (const char*)b + nb && (const char*)b < (const char*)a + na;
}

// Inputs and outputs in the same memory space: an address in one may alias the other.
bool same_side(int flags) { return !(flags & EDTB200_LABELS_ON_DEVICE) == !(flags & EDTB200_OUT_ON_DEVICE); }

int dispatch_first(int label_bytes, const void* labels, float* f, int64_t nlines, int64_t sx, float w,
                   int border, int flags, DeviceCache& dc, cudaStream_t s, const edtb200::XPlanes* planes = nullptr,
                   PlanesMarch* march = nullptr) {
  return with_label_width(label_bytes, [&](auto b) {
    return launch_first<b>(labels, f, nlines, sx, w, border, flags, planes, dc, s, march);
  });
}

int dispatch_later(int label_bytes, const void* labels, float* f, const edtb200::LineGeom& g, float w,
                   int lo, int hi, int flags, PassArith arith, DeviceCache& dc, cudaStream_t s, bool pdl,
                   const LaterNoise* planned = nullptr) {
  return with_label_width(label_bytes, [&](auto b) {
    return launch_later<b>(labels, planned, f, g, w, lo, hi, flags, arith, dc, s, pdl);
  });
}

// Grows a cached device buffer to at least `need` bytes; what it held is not kept.
template <class T>
cudaError_t grow(T*& p, size_t& have, size_t need) {
  if (have >= need) return cudaSuccess;
  if (p) cudaFree(p);
  p = nullptr; have = 0;
  const cudaError_t e = cudaMalloc(&p, need);
  if (e == cudaSuccess) have = need;
  return e;
}

// The residency contract of include/edt_b200.h for one call whose inputs and outputs may lie in
// host memory: open() probes the device, takes its host_call lock unless every buffer is on the
// device and picks the stream; in() / out() give the device address of each buffer, uploading a host
// input into the caller's staging buffer or noting a download from it; finish() runs the downloads
// in order and, when host memory is involved, waits for them.  The caller's current device is
// restored last, so the Scratch a call declares after its HostIO is freed while the call still
// holds the lock and the device.
struct HostIO {
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  bool in_dev = false, out_dev = false;
  cudaStream_t stream = nullptr;

  int open(int device, int flags, void* stream_v) {
    if (const int rc = probe(device, &dc)) return rc;
    in_dev = flags & EDTB200_LABELS_ON_DEVICE;
    out_dev = flags & EDTB200_OUT_ON_DEVICE;
    device_ = device;
    stream = static_cast<cudaStream_t>(stream_v);
    if (in_dev && out_dev) return 0;         // asynchronous on the caller's stream, no lock
    lock_ = std::unique_lock<std::mutex>(dc->host_call);
    // Both sides on the host and no stream given: the private stream.  With one side on the device
    // the legacy default stream (NULL) is kept: it is ordered after the work the caller queued on
    // the default / blocking streams that produced that buffer.
    if (!stream && !in_dev && !out_dev) {
      CUDA_TRY(private_stream(*dc));
      stream = dc->stream;
    }
    return 0;
  }
  template <class T>
  int in(const T* src, size_t bytes, void* staging, const T** dev) {
    *dev = in_dev ? src : static_cast<const T*>(staging);
    return in_dev ? 0 : upload(staging, src, bytes, device_, stream);
  }
  template <class T>
  T* out(T* dst, size_t bytes, T* staging) {
    if (out_dev) return dst;
    downloads_[count_++] = {dst, staging, bytes};
    return staging;
  }
  // in() / out() staged through the device's cached labels / distances buffer, grown for a host buffer
  template <class T>
  int in_labels(const T* src, size_t bytes, const T** dev) {
    if (!in_dev) CUDA_TRY(grow(dc->labels, dc->labels_bytes, bytes));
    return in(src, bytes, dc->labels, dev);
  }
  template <class T>
  int out_dist(T* dst, size_t bytes, T** dev) {
    if (!out_dev) CUDA_TRY(grow(dc->dist, dc->dist_bytes, bytes));
    *dev = out(dst, bytes, static_cast<T*>(static_cast<void*>(dc->dist)));
    return 0;
  }
  // out() staged through `scratch`, taken for a host buffer ("no device memory for <what>")
  template <class T>
  int out_staged(T* dst, size_t bytes, Scratch& scratch, const char* what, T** dev) {
    if (!out_dev)
      if (const int rc = scratch.take(*dc, bytes, stream, what)) return rc;
    *dev = out(dst, bytes, scratch.get<T>());
    return 0;
  }
  int finish() {
    for (int i = 0; i < count_; ++i) {
      const int rc = download(downloads_[i].dst, downloads_[i].src, downloads_[i].bytes, device_, stream);
      if (rc) return rc;
    }
    if (!(in_dev && out_dev)) CUDA_TRY(cudaStreamSynchronize(stream));
    return 0;
  }

 private:
  struct Download { void* dst; const void* src; size_t bytes; };
  Download downloads_[4];                    // at most the distances and three index planes
  int count_ = 0, device_ = 0;
  std::unique_lock<std::mutex> lock_;
};

// The label-noise plan of one transform (noise_plan) and the run-start planes that its X pass writes for
// its later passes (XPlanes): one bit per voxel and later axis, stream-ordered scratch freed on the
// stream when the owner goes out of scope.
struct RunPlanes {
  Scratch mem;
  edtb200::XPlanes x{};             // x.y null: none
  LaterNoise later[3];              // the later pass along axis k as planned (bits.start null: no plane)
  const edtb200::XPlanes* for_x() const { return x.y ? &x : nullptr; }
};

// The 32-bit words of the planes that plan np asks of transform t over `count` volumes (t.n[0], sy, sz):
// per later axis, the run-start plane (wpr = ceil(sx / 32) words per row), then the settled plane (one
// word per row); [y plane | settled_y | z plane | settled_z].
int64_t run_planes_words(const NoisePlan& np, const Transform& t, int64_t sy, int64_t sz, int64_t count) {
  const int64_t rows = sy * sz * count;
  return (rows * ((t.n[0] + 31) >> 5) + rows) * np.planes;
}

// Arms the later passes of rp as plan np says, with the planes (if any) laid out at p, run_planes_words
// of them.
void arm_run_planes(RunPlanes& rp, const NoisePlan& np, const Transform& t, uint32_t* p, int64_t sy, int64_t sz,
                    int64_t count) {
  for (int k = 1; k < 3; ++k) {
    rp.later[k].noise = np.noise;
    rp.later[k].plan = np.later[k];
  }
  if (!np.planes || !p) return;
  const int64_t sx = t.n[0], wpr = (sx + 31) >> 5, rows = sy * sz * count, words = rows * wpr;
  rp.x.sy = sy;
  rp.x.depth = sz;
  rp.x.y = p;
  rp.x.settled_y = p + words;
  rp.x.z = np.planes == 2 ? p + words + rows : nullptr;
  rp.x.settled_z = np.planes == 2 ? p + 2 * words + rows : nullptr;
  rp.x.ty = t.w[1] * t.w[1];         // the float products the later passes compare with (launch_later)
  rp.x.tz = np.planes == 2 ? t.w[2] * t.w[2] : 0.0f;
  // Y pass: outer = z (of every volume), inner = x; Z pass: outer = volume, inner = y * sx + x, rows
  // sy * wpr words apart.  Settled words: Y pass at z * sy + y, Z pass at volume * sz * sy + z * sy + y.
  if (np.reads[1])
    rp.later[1].bits = edtb200::RunBits{rp.x.y, wpr, sy * wpr, sx, wpr, np.later[1].settled ? rp.x.settled_y : nullptr,
                                        1, sy, np.refresh ? rp.x.settled_z : nullptr, np.refresh ? rp.x.tz : 0.0f,
                                        np.group[1]};
  if (np.reads[2])
    rp.later[2].bits = edtb200::RunBits{rp.x.z, sy * wpr, sz * sy * wpr, sx, wpr,
                                        np.later[2].settled ? rp.x.settled_z : nullptr, sy, sz * sy, nullptr, 0.0f,
                                        np.group[2]};
}

// Plans transform t over `count` volumes (t.n[0], sy, sz) laid end to end at labels / f, and takes the
// planes the plan asks for; where there is no room for them the later passes read the labels.
int take_run_planes(RunPlanes& rp, const Transform& t, const void* labels, const float* f, int64_t sy, int64_t sz,
                    int64_t count, DeviceCache& dc, cudaStream_t s) {
  const NoisePlan np = noise_plan(t, count, labels, f, dc);
  uint32_t* p = nullptr;
  if (np.planes) {
    if (rp.mem.alloc(dc, sizeof(uint32_t) * (size_t)run_planes_words(np, t, sy, sz, count), s) == cudaSuccess)
      p = rp.mem.get<uint32_t>();
    else
      cudaGetLastError();            // no room: the later passes read the labels
  }
  arm_run_planes(rp, np, t, p, sy, sz, count);
  return 0;
}

// The X pass over nlines rows; planes: the run-start planes it writes (null: none); march: the march
// of the plane-writing kernel asked for and launched (PlanesMarch, null: its own rule).
int x_pass(const Transform& t, const void* labels, float* f, int64_t nlines, DeviceCache& dc, cudaStream_t s,
           const RunPlanes* planes = nullptr, PlanesMarch* march = nullptr) {
  return dispatch_first(t.label_bytes, labels, f, nlines, t.n[0], t.w[0], t.border,
                        kernel_flags(t.flags, true, t.ndim == 1), dc, s, planes ? planes->for_x() : nullptr, march);
}

// The later pass along axis k over geometry g, with the borders lo / hi at the ends of its lines;
// planes: those its X pass wrote over the same volume (null: none).
int later_pass(const Transform& t, int k, const void* labels, float* f, const edtb200::LineGeom& g, int lo, int hi,
               DeviceCache& dc, cudaStream_t s, bool pdl, const RunPlanes* planes = nullptr) {
  return dispatch_later(t.label_bytes, labels, f, g, t.w[k], lo, hi, kernel_flags(t.flags, false, k == t.ndim - 1),
                        transform_arith(t.w, t.n, k), dc, s, pdl, planes ? &planes->later[k] : nullptr);
}

// Largest finite |f| (as float bits: non-negative floats order like their bits) and the exponent
// of the lowest set bit over all finite non-zero samples, for edtb200_pass_later, whose samples
// the host knows nothing about.  range = {0, 1024} on entry.
__global__ void __launch_bounds__(256) sample_range_kernel(const float* __restrict__ f, int64_t count,
                                                          int* range) {
  unsigned int hi = 0u;
  int low = 1024;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned int b = __float_as_uint(f[i]) & 0x7fffffffu;
    if (b >= 0x7f800000u || b == 0u) continue;           // +inf (and nan) are not sites; 0 has no bit
    hi = max(hi, b);
    const unsigned int e = b >> 23, m = (b & 0x7fffffu) | (e ? 0x800000u : 0u);
    low = min(low, (int)(e ? e : 1u) - 150 + (__ffs(m) - 1));
  }
  for (int o = 16; o; o >>= 1) {
    hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    low = min(low, __shfl_xor_sync(0xffffffffu, low, o));
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(reinterpret_cast<unsigned int*>(range), hi);
    atomicMin(range + 1, low);
  }
}

// Optional per-pass timing for bench.py: with profiling on, every transform of this thread records
// four CUDA events (before / between / after its axis passes) into a ring, so a timed loop can be
// analysed afterwards without any synchronisation inside it (edtb200_profile_passes /
// edtb200_pass_ms).
constexpr int kProfileRing = 256;
thread_local bool g_profile = false;
thread_local cudaEvent_t g_pass_events[kProfileRing][4];
thread_local bool g_pass_events_init = false;
thread_local int g_pass_marks[kProfileRing];       // highest mark index recorded in the slot
thread_local long g_pass_seq = 0;                  // transforms profiled so far

void mark_pass(int idx, cudaStream_t stream) {
  if (!g_profile) return;
  if (!g_pass_events_init) {
    for (auto& slot : g_pass_events) for (auto& e : slot) e = nullptr;
    g_pass_events_init = true;
  }
  if (idx == 0) ++g_pass_seq;
  const int slot = (int)((g_pass_seq - 1) % kProfileRing);
  cudaEvent_t& e = g_pass_events[slot][idx];
  if (!e && cudaEventCreate(&e) != cudaSuccess) { cudaGetLastError(); return; }
  cudaEventRecord(e, stream);
  g_pass_marks[slot] = idx;
}

// NVTX ranges edt.x / edt.y / edt.z / edt.halo.* (SURVEY.md section 5) around the launches, so
// that an Nsight Systems timeline names the passes.  libnvToolsExt is looked up at run time
// (dlopen), so it is not a dependency; without it the calls do nothing.
typedef int (*NvtxPushFn)(const char*);
typedef int (*NvtxPopFn)(void);
NvtxPushFn g_nvtx_push = nullptr;
NvtxPopFn g_nvtx_pop = nullptr;
std::once_flag g_nvtx_once;

void nvtx_init() {
  std::call_once(g_nvtx_once, [] {
    if (getenv("EDTB200_NO_NVTX")) return;
    const char* names[] = {"libnvToolsExt.so.1", "libnvToolsExt.so", nullptr};
    for (int i = 0; names[i]; ++i) {
      void* h = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
      if (!h) continue;
      g_nvtx_push = reinterpret_cast<NvtxPushFn>(dlsym(h, "nvtxRangePushA"));
      g_nvtx_pop = reinterpret_cast<NvtxPopFn>(dlsym(h, "nvtxRangePop"));
      if (g_nvtx_push && g_nvtx_pop) return;
      g_nvtx_push = nullptr; g_nvtx_pop = nullptr;
    }
  });
}
void nvtx_push(const char* name) { nvtx_init(); if (g_nvtx_push) g_nvtx_push(name); }
void nvtx_pop() { if (g_nvtx_pop) g_nvtx_pop(); }

// EDT_B200_VERBOSE=1: the calls report their device times on stderr, one "[edt_b200] ..." line each
// (SURVEY.md section 5).  A verbose call synchronises its stream to read them.
bool verbose() {
  static const bool on = getenv("EDT_B200_VERBOSE") != nullptr && atoi(getenv("EDT_B200_VERBOSE")) != 0;
  return on;
}

// The device times between the steps of one verbose call: stamp() after each step records an event on
// the stream, synchronize() waits for the last one, ms(a, b) is the time between stamps a and b (0 where
// an event is missing).  Off unless verbose(): no events, and synchronize() is false.  The events are
// destroyed on every exit.
class StepTimer {
 public:
  explicit StepTimer(cudaStream_t s) : s_(s) {}
  StepTimer(const StepTimer&) = delete;
  StepTimer& operator=(const StepTimer&) = delete;
  ~StepTimer() {
    if (!on_) return;
    for (int i = 0; i < n_; ++i)
      if (ev_[i]) cudaEventDestroy(ev_[i]);
    cudaGetLastError();
  }
  bool on() const { return on_; }
  void stamp() {
    if (!on_ || n_ == kMax) return;
    cudaEvent_t& e = ev_[n_++];
    if (cudaEventCreate(&e) != cudaSuccess) { e = nullptr; cudaGetLastError(); return; }
    if (cudaEventRecord(e, s_) != cudaSuccess) cudaGetLastError();
  }
  bool synchronize() const { return n_ > 0 && ev_[n_ - 1] && cudaEventSynchronize(ev_[n_ - 1]) == cudaSuccess; }
  float ms(int a, int b) const {
    float t = 0.0f;
    if (a < n_ && b < n_ && ev_[a] && ev_[b]) cudaEventElapsedTime(&t, ev_[a], ev_[b]);
    return t;
  }

 private:
  static constexpr int kMax = 6;
  cudaStream_t s_;
  bool on_ = verbose();
  int n_ = 0;
  cudaEvent_t ev_[kMax] = {};
};

// All passes of one transform on device-resident buffers: of `count` volumes of (sx, sy, sz) laid end
// to end, each transformed on its own with one launch per pass for all of them.  Every pass keeps one
// volume's extents for its arithmetic (transform_arith over t.n), so each volume gets the plan it
// would get alone.
int run_passes(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
               float wx, float wy, float wz, int border, int flags, float* f,
               DeviceCache& dc, cudaStream_t stream, int64_t count = 1) {
  const Transform t{label_bytes, ndim, flags, border, {wx, wy, wz}, {sx, sy, sz}};
  // The later passes are launched with programmatic stream serialization: the kernel before them
  // in the stream is our own previous pass, which never writes the labels, so their label staging
  // (before griddepcontrol.wait) may overlap its tail.  The per-axis entry points do not do this:
  // there the previous kernel is the caller's and may be the one producing the labels.
  // Every pass plans with one reading of the noise prediction (RunPlanes).  On predicted label noise
  // with wide labels the X pass also writes run-start bit planes, and the later passes read those
  // instead of the labels; a later pass reads its plane only after griddepcontrol.wait.
  RunPlanes planes;
  int rc = take_run_planes(planes, t, labels, f, sy, sz, count, dc, stream);
  if (rc) return rc;
  // verbose: per-pass device times of every transform, read from the mark_pass ring
  const bool profile_was = g_profile;
  if (verbose()) g_profile = true;
  mark_pass(0, stream);
  nvtx_push("edt.x");
  rc = x_pass(t, labels, f, sy * sz * count, dc, stream, &planes);
  nvtx_pop();
  mark_pass(1, stream);
  if (!rc && ndim >= 2) {
    nvtx_push("edt.y");
    rc = later_pass(t, 1, labels, f, geom_for_axis(1, sx, sy, sz, count), border, border, dc, stream, /*pdl=*/true,
                    &planes);
    nvtx_pop();
    mark_pass(2, stream);
  }
  if (!rc && ndim >= 3) {
    nvtx_push("edt.z");
    rc = later_pass(t, 2, labels, f, geom_for_axis(2, sx, sy, sz, count), border, border, dc, stream, /*pdl=*/true,
                    &planes);
    nvtx_pop();
    mark_pass(3, stream);
  }
  if (verbose()) {
    g_profile = profile_was;
    float ms[3] = {0.0f, 0.0f, 0.0f};
    if (!rc && edtb200_pass_ms(0, ms) == 0) {
      const double nvox = (double)sx * (double)sy * (double)sz * (double)count;
      const double total = ms[0] + ms[1] + ms[2];
      fprintf(stderr, "[edt_b200] %lldx%lldx%lld L=%d  x %.3f ms  y %.3f ms  z %.3f ms  total %.3f ms  "
                      "%.0f Mvox/s  %.0f GB/s algorithmic\n",
              (long long)sx, (long long)sy, (long long)sz, label_bytes, ms[0], ms[1], ms[2], total,
              total > 0 ? nvox / total / 1e3 : 0.0,
              total > 0 ? nvox * (3.0 * label_bytes + 20.0) / total / 1e6 : 0.0);
    }
  }
  return rc;
}

// The parabolic passes (dilate: dilation) along every axis of `count` volumes of (sx, sy, sz) laid end
// to end: the first from `in` into `out`, the others in place on `out`; codes[k] non-null: pass k also
// writes its site codes there.  kernel[k] is what pass k ran (launch_parabolic_pass), -1 for none; the
// timer is stamped after each pass.
int parabolic_passes(const float* in, float* out, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                     const float w[3], bool dilate, int* const codes[3], int kernel[3], StepTimer& timer,
                     DeviceCache& dc, cudaStream_t s) {
  kernel[0] = kernel[1] = kernel[2] = -1;
  int rc = 0;
  for (int k = 0; !rc && k < ndim; ++k) {
    edtb200::LineGeom g = geom_for_axis(k, sx, sy, sz, count);
    if (k == 0) {                              // rows of sx contiguous samples
      g.outer_count = sy * sz * count; g.outer_stride = sx; g.inner_count = 1; g.line_stride = 1; g.n = (int)sx;
    }
    rc = launch_parabolic_pass(k == 0 ? in : out, out, g, k == 0, w[k], dilate, dc, s, &kernel[k], codes[k]);
    timer.stamp();
  }
  return rc;
}

// All passes of one bounded transform (include/edt_b200.h) on device-resident buffers: the X pass,
// then each later pass in the window kernel where bp says so (out of place) and in launch_later
// otherwise (in place, without its sqrt / sign), then -- unless the last pass was a window pass,
// which cuts in its store -- the cut.  The X pass writes f or one scratch volume, whichever makes the
// last window pass that writes distances land in f.  `count` volumes of (sx, sy, sz) laid end to end
// are transformed each on its own, as run_passes does.  sel: a morphology step (edt_morphology.cuh),
// whose last store writes sel's labels or mask instead of distances -- in the last pass where it takes
// the window kernel, else in the select that replaces the cut (f then holds scratch distances).
int run_bounded_passes(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                       float wx, float wy, float wz, int border, int flags, float* f, const BoundedPlan& bp,
                       DeviceCache& dc, cudaStream_t s, int64_t count = 1, const edtb200::MorphSelect* sel = nullptr) {
  const Transform t{label_bytes, ndim, flags, border, {wx, wy, wz}, {sx, sy, sz}};
  const int64_t total = sx * sy * sz * count;
  int windows = 0;                                // window passes that write distances
  for (int k = 1; k < ndim; ++k) windows += bp.windowed[k] && !(sel && k == ndim - 1) ? 1 : 0;
  Scratch other;
  if (windows)
    if (const int rc = other.take(dc, sizeof(float) * (size_t)total, s, "the bounded transform's scratch volume"))
      return rc;
  float* buf[2] = {f, other.get<float>()};
  int cur = windows % 2;
  int rc = dispatch_first(label_bytes, labels, buf[cur], sy * sz * count, sx, wx, border,
                          kernel_flags(flags, true, false), dc, s);
  for (int k = 1; !rc && k < ndim; ++k) {
    const edtb200::LineGeom g = geom_for_axis(k, sx, sy, sz, count);
    const PassArith arith = transform_arith(t.w, t.n, k);
    if (bp.windowed[k] && sel && k == ndim - 1) {
      rc = launch_window_select(labels, label_bytes, buf[cur], g, t.w[k], (int)bp.radius[k], border, border, arith,
                                bp.bound, *sel, dc, s);
    } else if (bp.windowed[k]) {
      rc = with_label_width(label_bytes, [&](auto b) {
        return launch_later_window<b>(labels, buf[cur], buf[cur ^ 1], nullptr, g, t.w[k], (int)bp.radius[k], border,
                                      border, kernel_flags(flags, false, k == ndim - 1), arith, bp.bound, dc, s);
      });
      cur ^= 1;
    } else {
      rc = dispatch_later(label_bytes, labels, buf[cur], g, t.w[k], border, border, 0, arith, dc, s, /*pdl=*/false);
    }
  }
  if (rc || (ndim >= 2 && bp.windowed[ndim - 1])) return rc;
  if (sel) return launch_morph_select(f, total, bp.bound, *sel, dc, s);
  return with_label_width(label_bytes, [&](auto b) {
    return launch_bounded_cut<b>(labels, f, nullptr, total, bp.bound, kernel_flags(flags, false, true), dc, s);
  });
}

// All passes of one feature transform on device-resident buffers: the site-tracking passes, out of
// place and alternating between `dist` and one scratch volume so that the last lands in `dist`, then
// the resolver.  dist may be null (the distances then stay in scratch).  `count` volumes of
// (sx, sy, sz) laid end to end are transformed each on its own, as run_passes does; the index planes
// hold coordinates within each voxel's own volume.  bp: a bounded feature transform (count 1), whose
// later passes take the window kernel where it says so; when the last pass does not, that pass runs
// without its sqrt / sign and the cut follows it, on the distances and the last pass's codes.
int run_feature_passes(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                       float wx, float wy, float wz, int border, int flags, float* dist, int32_t* const idx[3],
                       DeviceCache& dc, cudaStream_t s, int64_t count = 1, const BoundedPlan* bp = nullptr) {
  const Transform t{label_bytes, ndim, flags, border, {wx, wy, wz}, {sx, sy, sz}};
  const size_t total = (size_t)(sx * sy * sz * count);
  Scratch own_dist, other, codes;
  auto take = [&](Scratch& sc, size_t bytes) {
    if (sc.alloc(dc, bytes, s) == cudaSuccess) return 0;
    cudaGetLastError();
    return fail(EDTB200_ENOMEM, "no device memory for the feature transform's scratch (%zu bytes)", bytes);
  };
  int rc = dist ? 0 : take(own_dist, total * sizeof(float));
  if (!rc && ndim >= 2) rc = take(other, total * sizeof(float));
  if (!rc) rc = take(codes, (size_t)ndim * total * sizeof(int));
  if (rc) return rc;
  float* buf[2] = {dist ? dist : own_dist.get<float>(), other.get<float>()};
  int* code_planes[3] = {nullptr, nullptr, nullptr};
  for (int k = 0; k < ndim; ++k) code_planes[k] = codes.get<int>() + (size_t)k * total;
  // pass k writes buf[(ndim - 1 - k) % 2]: the last one (k = ndim - 1) writes buf[0]
  const bool cut = bp && !(ndim >= 2 && bp->windowed[ndim - 1]);
  rc = with_label_width(label_bytes, [&](auto b) {
    return launch_first_sites<b>(labels, buf[(ndim - 1) % 2], code_planes[0], sy * sz * count, sx, wx, border,
                                 kernel_flags(flags, true, ndim == 1 && !cut), dc, s);
  });
  for (int k = 1; !rc && k < ndim; ++k) {
    const int kflags = kernel_flags(flags, false, k == ndim - 1 && !cut);
    rc = with_label_width(label_bytes, [&](auto b) {
      if (bp && bp->windowed[k])
        return launch_later_window<b>(labels, buf[(ndim - k) % 2], buf[(ndim - 1 - k) % 2], code_planes[k],
                                      geom_for_axis(k, sx, sy, sz, count), t.w[k], (int)bp->radius[k], border,
                                      border, kflags, transform_arith(t.w, t.n, k), bp->bound, dc, s);
      return launch_later_sites<b>(labels, buf[(ndim - k) % 2], buf[(ndim - 1 - k) % 2], code_planes[k],
                                   geom_for_axis(k, sx, sy, sz, count), t.w[k], border, border, kflags,
                                   transform_arith(t.w, t.n, k), dc, s);
    });
  }
  if (!rc && cut)
    rc = with_label_width(label_bytes, [&](auto b) {
      return launch_bounded_cut<b>(labels, buf[0], code_planes[ndim - 1], (int64_t)total, bp->bound,
                                   kernel_flags(flags, false, true), dc, s);
    });
  if (rc) return rc;
  return with_label_width(label_bytes, [&](auto b) {
    return launch_resolve_sites<b>(labels, code_planes, ndim, sx, sy, sz, count, !(flags & EDTB200_SIGNED), idx, dc,
                                   s);
  });
}

// The steps of a two-slot pipeline over `count` items: each gets the item, its slot (k % 2) and the
// stream to queue on.  `item` names an item in error messages ("volume", "chunk").  upload_writes_results:
// the upload also fills the buffer the download reads (the passes work in place on uploaded data).
struct PipelineSteps {
  const char* item = "item";
  bool upload_writes_results = false;
  std::function<int(int k, int slot, cudaStream_t)> upload, passes, download;
};

// The device's three pipeline streams (uploads, passes = the private stream, downloads) and the
// events that order the two slots; created on first use by the holder of host_call.
int pipeline_streams(DeviceCache& dc) {
  CUDA_TRY(private_stream(dc));
  if (!dc.stream_up) CUDA_TRY(cudaStreamCreateWithFlags(&dc.stream_up, cudaStreamNonBlocking));
  if (!dc.stream_down) CUDA_TRY(cudaStreamCreateWithFlags(&dc.stream_down, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    if (!dc.ev_up[i]) CUDA_TRY(cudaEventCreateWithFlags(&dc.ev_up[i], cudaEventDisableTiming));
    if (!dc.ev_comp[i]) CUDA_TRY(cudaEventCreateWithFlags(&dc.ev_comp[i], cudaEventDisableTiming));
    if (!dc.ev_down[i]) CUDA_TRY(cudaEventCreateWithFlags(&dc.ev_down[i], cudaEventDisableTiming));
  }
  return 0;
}

// Runs the steps of items 0..count-1 through two device slots, the caller holding host_call.  Item k
// uses slot k % 2.  Three streams: uploads (fed by a helper thread, so that pageable buffers can be
// staged in both directions at once), the passes, downloads (this thread).
//   upload k    waits for the passes of k-2 (they read the slot's inputs), and with
//               upload_writes_results for download k-2 as well (it reads what the upload overwrites)
//   passes k    wait for upload k and for download k-2 (it reads the slot's results)
//   download k  waits for the passes of k
// Host-side counters make sure an event has been RECORDED before someone waits on it.  Returns when
// every download has landed; after a failure, once the helper thread has ended and every stream is
// idle.
int run_pipeline(DeviceCache& dc, int device, int count, const PipelineSteps& steps) {
  int rc = pipeline_streams(dc);
  if (rc) return rc;
  std::mutex m;
  std::condition_variable cv;
  int uploads_queued = 0, passes_queued = 0, downloads_queued = 0, failed = 0;
  char upload_error[sizeof(g_error)] = "";
  std::thread uploader([&] {
    cudaSetDevice(device);
    for (int k = 0; k < count; ++k) {
      const int slot = k & 1;
      int urc = 0;
      if (k >= 2) {
        std::unique_lock<std::mutex> l(m);
        cv.wait(l, [&] {
          return (passes_queued >= k - 1 && (!steps.upload_writes_results || downloads_queued >= k - 1)) || failed;
        });
        if (failed) return;
        if (cudaStreamWaitEvent(dc.stream_up, dc.ev_comp[slot], 0) != cudaSuccess) urc = EDTB200_ECUDA;
        if (!urc && steps.upload_writes_results && cudaStreamWaitEvent(dc.stream_up, dc.ev_down[slot], 0) != cudaSuccess)
          urc = EDTB200_ECUDA;
      }
      if (!urc) urc = steps.upload(k, slot, dc.stream_up);
      if (!urc && cudaEventRecord(dc.ev_up[slot], dc.stream_up) != cudaSuccess) urc = EDTB200_ECUDA;
      std::lock_guard<std::mutex> l(m);
      if (urc) {
        failed = urc;
        snprintf(upload_error, sizeof(upload_error), "upload of %s %d failed: %.400s", steps.item, k,
                 urc == EDTB200_ECUDA ? cudaGetErrorString(cudaGetLastError()) : g_error);
      } else {
        uploads_queued = k + 1;
      }
      cv.notify_all();
      if (urc) return;
    }
  });
  auto bail = [&](int code) {
    { std::lock_guard<std::mutex> l(m); if (!failed) failed = code; }
    cv.notify_all();
    uploader.join();
    cudaStreamSynchronize(dc.stream_up); cudaStreamSynchronize(dc.stream); cudaStreamSynchronize(dc.stream_down);
    return code;
  };
  #define PIPE_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { \
      fail(EDTB200_ECUDA, "%s: %s", #expr, cudaGetErrorString(e_)); return bail(EDTB200_ECUDA); } } while (0)
  for (int k = 0; k < count; ++k) {
    const int slot = k & 1;
    {
      std::unique_lock<std::mutex> l(m);
      cv.wait(l, [&] { return uploads_queued >= k + 1 || failed; });
      if (failed) { l.unlock(); uploader.join(); cudaDeviceSynchronize(); return fail(failed, "%s", upload_error); }
    }
    PIPE_TRY(cudaStreamWaitEvent(dc.stream, dc.ev_up[slot], 0));
    if (k >= 2) PIPE_TRY(cudaStreamWaitEvent(dc.stream, dc.ev_down[slot], 0));
    rc = steps.passes(k, slot, dc.stream);
    if (rc) return bail(rc);
    PIPE_TRY(cudaEventRecord(dc.ev_comp[slot], dc.stream));
    { std::lock_guard<std::mutex> l(m); passes_queued = k + 1; }
    cv.notify_all();
    PIPE_TRY(cudaStreamWaitEvent(dc.stream_down, dc.ev_comp[slot], 0));
    rc = steps.download(k, slot, dc.stream_down);
    if (rc) return bail(rc);
    PIPE_TRY(cudaEventRecord(dc.ev_down[slot], dc.stream_down));
    { std::lock_guard<std::mutex> l(m); downloads_queued = k + 1; }
    cv.notify_all();
  }
  #undef PIPE_TRY
  uploader.join();
  CUDA_TRY(cudaStreamSynchronize(dc.stream_down));
  return 0;
}

}  // namespace

extern "C" {

int edtb200_version(void) { return EDTB200_VERSION; }

const char* edtb200_last_error(void) { return g_error; }

int edtb200_device_count(void) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess) { cudaGetLastError(); return 0; }
  return count;
}

int edtb200_transform(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                      float wx, float wy, float wz, int black_border, int flags, float* out,
                      int device, void* stream_v) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  const int64_t total = sx * sy * sz;
  if (total == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const void* d_labels = nullptr;
  float* d_out = nullptr;
  if ((rc = io.in_labels(labels, (size_t)total * (size_t)label_bytes, &d_labels)) ||
      (rc = io.out_dist(out, (size_t)total * sizeof(float), &d_out)))
    return rc;
  rc = run_passes(d_labels, label_bytes, ndim, sx, sy, sz, wx, wy, wz, black_border != 0, flags, d_out, *io.dc,
                  io.stream);
  return rc ? rc : io.finish();
}

int edtb200_feature_transform(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                              float wx, float wy, float wz, int black_border, int flags, float* dist_out,
                              int32_t* const* idx_out, int device, void* stream_v) {
  return edtb200_feature_transform_stack(labels, label_bytes, ndim, sx, sy, sz, 1, wx, wy, wz, black_border, flags,
                                         dist_out, idx_out, device, stream_v);
}

int edtb200_transform_batch(const void* const* labels, float* const* outs, int count, int label_bytes, int ndim,
                            int64_t sx, int64_t sy, int64_t sz, float wx, float wy, float wz,
                            int black_border, int flags, int device) {
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (flags & (EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_transform_batch pipelines HOST buffers; device-resident volumes are "
                                "already asynchronous through edtb200_transform");
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  const int64_t total = sx * sy * sz;
  if (total == 0 || count == 0) return 0;
  if (!labels || !outs) return fail(EDTB200_EINVAL, "null pointer");
  for (int k = 0; k < count; ++k)
    if (!labels[k] || !outs[k]) return fail(EDTB200_EINVAL, "null pointer in volume %d", k);

  DeviceGuard restore_device;
  DeviceCache* dcp = nullptr;
  rc = probe(device, &dcp);
  if (rc) return rc;
  DeviceCache& dc = *dcp;
  std::lock_guard<std::mutex> host_call(dc.host_call);
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, out_bytes = (size_t)total * sizeof(float);
  CUDA_TRY(grow(dc.labels, dc.labels_bytes, lab_bytes));
  CUDA_TRY(grow(dc.dist, dc.dist_bytes, out_bytes));
  if (count > 1) {
    CUDA_TRY(grow(dc.labels2, dc.labels2_bytes, lab_bytes));
    CUDA_TRY(grow(dc.dist2, dc.dist2_bytes, out_bytes));
  }
  void* d_labels[2] = {dc.labels, dc.labels2};
  float* d_dist[2] = {dc.dist, dc.dist2};
  const int border = black_border != 0;
  PipelineSteps steps;
  steps.item = "volume";
  steps.upload = [&](int k, int slot, cudaStream_t s) { return upload(d_labels[slot], labels[k], lab_bytes, device, s); };
  steps.passes = [&](int, int slot, cudaStream_t s) {
    return run_passes(d_labels[slot], label_bytes, ndim, sx, sy, sz, wx, wy, wz, border, flags, d_dist[slot], dc, s);
  };
  steps.download = [&](int k, int slot, cudaStream_t s) { return download(outs[k], d_dist[slot], out_bytes, device, s); };
  return run_pipeline(dc, device, count, steps);
}

}  // extern "C"

// ---- one host volume larger than the device, streamed through it in chunks -------------------
namespace {

// One phase of edtb200_transform_chunked / edtb200_feature_transform_chunked (the plans of
// include/edt_b200.h): `extent` slices of `slice_vox` voxels and `slice_bytes` device bytes each, in
// `count` chunks of at most `most` slices (count 0: the budget is below `need`, the least that works).
struct PhasePlan {
  int64_t extent = 0, slice_vox = 0, count = 0, most = 0;
  size_t slice_bytes = 0, need = 0;
  int64_t start(int64_t k) const { return extent * k / count; }        // chunk sizes differ by one at most
  int64_t size(int64_t k) const { return start(k + 1) - start(k); }
};

// Frees this device's cached whole-volume buffers and trims its private pool (the caller holds
// host_call), so that a chunked call after a one-shot call that ran out of memory finds it free.
void drop_volume_buffers(DeviceCache& dc) {
  void* bufs[] = {dc.labels, dc.dist, dc.labels2, dc.dist2};
  for (void* b : bufs) if (b) cudaFree(b);
  dc.labels = dc.labels2 = nullptr; dc.dist = dc.dist2 = nullptr;
  dc.labels_bytes = dc.labels2_bytes = dc.dist_bytes = dc.dist2_bytes = 0;
  if (dc.pool) cudaMemPoolTrimTo(dc.pool, 0);
  cudaGetLastError();
}

// The slots of one phase: labels, then `planes` volumes of 4 bytes per voxel (distances, site codes,
// coordinates), in one scratch allocation each.
struct ChunkSlots {
  Scratch buf[2];
  void* labels[2] = {nullptr, nullptr};
  size_t lab = 0, vox = 0;
  // volume j of slot `slot`
  template <class T = float>
  T* plane(int slot, int j) const { return reinterpret_cast<T*>(buf[slot].get<char>() + lab + (size_t)j * vox * 4); }
};

// Runs the chunks of plan p through run_pipeline; fill(slots, steps) sets the steps, which work on
// the phase's slots of label_bytes and `planes` volumes.  The slots are taken on dc.stream and freed
// on it when the phase returns, so that a next phase's slots reuse their memory instead of competing
// with them for the budget.  Returns when every download has landed.
template <class Fill>
int run_phase(DeviceCache& dc, int device, const PhasePlan& p, int label_bytes, int planes, Fill fill) {
  if (const int rc = pipeline_streams(dc)) return rc;   // dc.stream, which the slots are taken on
  ChunkSlots slots;
  slots.vox = (size_t)p.most * (size_t)p.slice_vox;
  slots.lab = (slots.vox * (size_t)label_bytes + 255) & ~size_t(255);
  const size_t bytes = slots.lab + (size_t)planes * slots.vox * 4;
  for (int i = 0; i < (p.count > 1 ? 2 : 1); ++i) {
    if (slots.buf[i].alloc(dc, bytes, dc.stream) != cudaSuccess) {
      cudaGetLastError();
      return fail(EDTB200_ENOMEM, "no device memory for a chunk slot of %zu bytes: give a smaller device_bytes", bytes);
    }
    slots.labels[i] = slots.buf[i].get();
  }
  CUDA_TRY(cudaStreamSynchronize(dc.stream));   // allocated on the passes' stream, used on all three
  PipelineSteps steps;
  fill(slots, steps);
  return run_pipeline(dc, device, (int)p.count, steps);
}

// A host buffer of a streaming call; `written`: the call writes it.
struct HostRange { const void* p; size_t bytes; const char* name; bool written; };

// Fails with "<a> and <b> overlap" on the first pair, in list order, of non-null buffers that share a
// byte where the call writes at least one of the two (inputs may overlap each other).
int check_overlap(std::initializer_list<HostRange> ranges) {
  for (const HostRange* a = ranges.begin(); a != ranges.end(); ++a)
    for (const HostRange* b = a + 1; b != ranges.end(); ++b) {
      const char *pa = static_cast<const char*>(a->p), *pb = static_cast<const char*>(b->p);
      if (pa && pb && (a->written || b->written) && pa < pb + b->bytes && pb < pa + a->bytes)
        return fail(EDTB200_EINVAL, "%s and %s overlap", a->name, b->name);
    }
  return 0;
}

// A call that streams host buffers through `device`, as HostIO serves a one-shot call: the caller's
// current device is restored on return, and from lock() on the call holds the device's host_call
// lock and its device budget: `device_bytes`, or with 0 the memory free once the device's cached
// whole-volume buffers are dropped, less EDTB200_CHUNK_RESERVE.  The buffers are dropped either way.
struct StreamingCall {
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  size_t budget = 0;

  int open(int device) { return probe(device, &dc); }
  int lock(size_t device_bytes) {
    lock_ = std::unique_lock<std::mutex>(dc->host_call);
    drop_volume_buffers(*dc);
    budget = device_bytes;
    if (device_bytes == 0) {
      size_t free_bytes = 0, total_bytes = 0;
      CUDA_TRY(cudaMemGetInfo(&free_bytes, &total_bytes));
      budget = free_bytes > EDTB200_CHUNK_RESERVE ? free_bytes - EDTB200_CHUNK_RESERVE : 0;
    }
    return 0;
  }
  // A phase within the budget: extent slices of slice_vox voxels that cost voxel_bytes device bytes
  // per voxel each (a slot's buffers and the phase's per-launch scratch); a chunk holds at most `cap`
  // slices.
  PhasePlan plan(int64_t extent, int64_t slice_vox, size_t voxel_bytes, int64_t cap) const {
    PhasePlan p;
    p.extent = extent;
    p.slice_vox = slice_vox;
    p.slice_bytes = (size_t)slice_vox * voxel_bytes;
    p.need = (size_t)(extent < 2 ? extent : 2) * p.slice_bytes;
    if (extent <= cap && (size_t)extent <= budget / p.slice_bytes) {
      p.count = 1;
    } else {
      const int64_t c = std::min<int64_t>(cap, (int64_t)(budget / (2 * p.slice_bytes)));
      if (c == 0) return p;
      p.count = (extent + c - 1) / c;
    }
    p.most = (extent + p.count - 1) / p.count;
    return p;
  }

 private:
  std::unique_lock<std::mutex> lock_;
};

// The two phases of a chunked transform of an (sx, sy, sz) volume.  Phase 1 cuts the last axis (z
// slabs in 3-D, row ranges in 2-D) into slices of `plane` voxels; phase 2 cuts the axis before it
// into boxes of whole lines along the last axis, slices of `unit` voxels per index of the last axis
// and `line_vox` in all.
struct TwoPhase {
  int64_t n_last, n_cut, unit, plane, line_vox;
  PhasePlan p1, p2;

  TwoPhase(int ndim, int64_t sx, int64_t sy, int64_t sz)
      : n_last(ndim == 3 ? sz : sy), n_cut(ndim == 3 ? sy : sx), unit(ndim == 3 ? sx : 1), plane(unit * n_cut),
        line_vox(unit * n_last) {}

  // Plans both phases within the call's budget from their device bytes per voxel and the most slices
  // of a phase-2 chunk, and reports the chunk counts; `what` names the transform where the budget
  // cannot hold one chunk.
  int plan(const StreamingCall& call, size_t voxel_bytes1, size_t voxel_bytes2, int64_t cap2, const char* what,
           int64_t* chunks) {
    p1 = call.plan(n_last, plane, voxel_bytes1, n_last);
    p2 = call.plan(n_cut, line_vox, voxel_bytes2, cap2);
    if (p1.count == 0 || p2.count == 0)
      return fail(EDTB200_ENOMEM, "a device budget of %zu bytes cannot hold one chunk: the chunked %s needs at "
                                  "least %zu bytes", call.budget, what, std::max(p1.need, p2.need));
    if (chunks) { chunks[0] = p1.count; chunks[1] = p2.count; }
    return 0;
  }

  // Chunk k of a host volume of `bytes` per voxel.  Phase 1: size(k) whole slices, one range.
  HostBox slab(const void* base, int64_t k, size_t bytes) const {
    const size_t n = (size_t)(p1.size(k) * plane) * bytes;
    return HostBox{host(base) + (size_t)(p1.start(k) * plane) * bytes, n, n, 1};
  }
  // Phase 2: n_last rows of size(k) * unit voxels, one per index along the last axis, `plane` voxels
  // apart.
  HostBox lines(const void* base, int64_t k, size_t bytes) const {
    return HostBox{host(base) + (size_t)(p2.start(k) * unit) * bytes, (size_t)(p2.size(k) * unit) * bytes,
                   (size_t)plane * bytes, (size_t)n_last};
  }
  static char* host(const void* base) { return static_cast<char*>(const_cast<void*>(base)); }
};

}  // namespace

extern "C" {

int edtb200_transform_chunked(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                              float wx, float wy, float wz, int black_border, int flags, float* out,
                              int device, size_t device_bytes, int64_t* chunks) {
  if (chunks) chunks[0] = chunks[1] = 0;
  if (flags & (EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_transform_chunked streams HOST buffers through the device; a volume on "
                                "the device fits it: use edtb200_transform");
  if (ndim != 2 && ndim != 3)
    return fail(EDTB200_EINVAL, "edtb200_transform_chunked needs a 2-D or 3-D volume (got ndim %d)", ndim);
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  const int64_t total = sx * sy * sz;
  if (total == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, out_bytes = (size_t)total * sizeof(float);
  if ((rc = check_overlap({{labels, lab_bytes, "labels", false}, {out, out_bytes, "out", true}}))) return rc;

  StreamingCall call;
  if ((rc = call.open(device)) || (rc = call.lock(device_bytes))) return rc;
  DeviceCache& dc = *call.dc;

  // Phase 1 cuts the last axis: X pass, and in 3-D the Y pass.  Phase 2 cuts the axis before it: the
  // last pass.
  const int border = black_border != 0;
  const Transform t{label_bytes, ndim, flags, border, {wx, wy, wz}, {sx, sy, sz}};
  const int last = ndim - 1;
  TwoPhase two(ndim, sx, sy, sz);
  const int64_t cap2 = std::max<int64_t>(1, (int64_t)((((int64_t)1 << 32) - 65) / two.line_vox));
  const bool long1 = ndim == 3 && later_pass_is_long(geom_for_axis(1, sx, sy, sz), transform_arith(t.w, t.n, 1),
                                                     dc.max_smem_optin);
  const int64_t c2 = std::min(two.n_cut, cap2);
  const edtb200::LineGeom g2 = ndim == 3 ? geom_for_axis(2, sx, c2, sz) : geom_for_axis(1, c2, sy, 1);
  const bool long2 = later_pass_is_long(g2, transform_arith(t.w, t.n, last), dc.max_smem_optin);
  // per voxel: the labels and the distances, and the long-line kernel's two scratch volumes
  if ((rc = two.plan(call, label_bytes + 4 + (long1 ? 8 : 0), label_bytes + 4 + (long2 ? 8 : 0), cap2, "transform",
                     chunks)))
    return rc;

  const auto t0 = std::chrono::steady_clock::now();
  rc = run_phase(dc, device, two.p1, label_bytes, 1, [&](const ChunkSlots& slots, PipelineSteps& steps) {
    steps.item = "phase-1 chunk";
    steps.upload = [&](int k, int slot, cudaStream_t s) {
      return upload_box(slots.labels[slot], two.slab(labels, k, label_bytes), device, s);
    };
    steps.passes = [&](int k, int slot, cudaStream_t s) {
      int r = x_pass(t, slots.labels[slot], slots.plane(slot, 0), two.plane / sx * two.p1.size(k), dc, s);
      if (!r && ndim == 3)                                  // behind our own X pass
        r = later_pass(t, 1, slots.labels[slot], slots.plane(slot, 0), geom_for_axis(1, sx, sy, two.p1.size(k)),
                       border, border, dc, s, /*pdl=*/true);
      return r;
    };
    steps.download = [&](int k, int slot, cudaStream_t s) {
      return download_box(two.slab(out, k, sizeof(float)), slots.plane(slot, 0), device, s);
    };
  });
  if (rc) return rc;
  const auto t1 = std::chrono::steady_clock::now();
  rc = run_phase(dc, device, two.p2, label_bytes, 1, [&](const ChunkSlots& slots, PipelineSteps& steps) {
    steps.item = "phase-2 chunk";
    steps.upload_writes_results = true;            // the intermediate distances go up into the slot
    steps.upload = [&](int k, int slot, cudaStream_t s) {
      int r = upload_box(slots.labels[slot], two.lines(labels, k, label_bytes), device, s);
      return r ? r : upload_box(slots.plane(slot, 0), two.lines(out, k, sizeof(float)), device, s);
    };
    steps.passes = [&](int k, int slot, cudaStream_t s) {
      const int64_t c = two.p2.size(k);
      const edtb200::LineGeom g = ndim == 3 ? geom_for_axis(2, sx, c, sz) : geom_for_axis(1, c, sy, 1);
      return later_pass(t, last, slots.labels[slot], slots.plane(slot, 0), g, border, border, dc, s, /*pdl=*/false);
    };
    steps.download = [&](int k, int slot, cudaStream_t s) {
      return download_box(two.lines(out, k, sizeof(float)), slots.plane(slot, 0), device, s);
    };
  });
  if (rc) return rc;
  if (verbose()) {
    const auto t2 = std::chrono::steady_clock::now();
    const double ms1 = std::chrono::duration<double, std::milli>(t1 - t0).count();
    const double ms2 = std::chrono::duration<double, std::milli>(t2 - t1).count();
    fprintf(stderr, "[edt_b200] chunked %lldx%lldx%lld L=%d  budget %zu  chunks %lld + %lld  up %.3f GB  down %.3f GB  "
                    "phase 1 %.1f ms  phase 2 %.1f ms\n",
            (long long)sx, (long long)sy, (long long)sz, label_bytes, call.budget, (long long)two.p1.count,
            (long long)two.p2.count, (2.0 * label_bytes + 4.0) * (double)total / 1e9, 8.0 * (double)total / 1e9, ms1,
            ms2);
  }
  return 0;
}

int edtb200_feature_transform_chunked(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy,
                                      int64_t sz, float wx, float wy, float wz, int black_border, int flags,
                                      float* dist_out, int32_t* const* idx_out, int device, size_t device_bytes,
                                      int64_t* chunks) {
  if (chunks) chunks[0] = chunks[1] = 0;
  if (flags & (EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_feature_transform_chunked streams HOST buffers through the device; a volume "
                                "on the device fits it: use edtb200_feature_transform");
  if (ndim != 2 && ndim != 3)
    return fail(EDTB200_EINVAL, "edtb200_feature_transform_chunked needs a 2-D or 3-D volume (got ndim %d)", ndim);
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  const int64_t total = sx * sy * sz;
  if (total == 0) return 0;
  if (!labels || !idx_out) return fail(EDTB200_EINVAL, "null pointer");
  for (int k = 0; k < ndim; ++k)
    if (!idx_out[k]) return fail(EDTB200_EINVAL, "null index plane %d", k);
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, vol_bytes = (size_t)total * sizeof(float);
  if ((rc = check_overlap({{labels, lab_bytes, "labels", false}, {dist_out, vol_bytes, "dist_out", true},
                           {idx_out[0], vol_bytes, "index plane 0", true},
                           {idx_out[1], vol_bytes, "index plane 1", true},
                           {ndim == 3 ? idx_out[2] : nullptr, vol_bytes, "index plane 2", true}})))
    return rc;

  StreamingCall call;
  if ((rc = call.open(device)) || (rc = call.lock(device_bytes))) return rc;
  DeviceCache& dc = *call.dc;

  // The phases of edtb200_transform_chunked, on the site-tracking passes.  Phase 1 resolves every
  // voxel's site within its slice (3-D: (qx, qy); 2-D: the X code, qx), phase 2 follows the last
  // axis's code to the partial site on the voxel's own line, which lies in the same chunk.
  const int border = black_border != 0;
  const bool zero_bg = !(flags & EDTB200_SIGNED);
  const Transform t{label_bytes, ndim, flags, border, {wx, wy, wz}, {sx, sy, sz}};
  const int last = ndim - 1;
  TwoPhase two(ndim, sx, sy, sz);
  // Slot volumes (4 bytes per voxel each) beside the labels:
  //   phase 1, 3-D  0 X distances, then qx; 1 Y distances; 2 X codes; 3 Y codes, then qy
  //   phase 1, 2-D  0 X distances; 1 X codes (= qx)
  //   phase 2       0 intermediate distances, then x; 1 distances; 2 qx; 3 qy (3-D); `codes` the last
  //                 axis's codes, then its coordinate; 5 y (3-D)
  // and per launch of a later pass the long-line kernel's hull, 4 bytes per voxel of the chunk.
  const int planes1 = ndim == 3 ? 4 : 2, planes2 = ndim == 3 ? 6 : 4, codes = ndim == 3 ? 4 : 3;
  if ((rc = two.plan(call, label_bytes + 4 * planes1 + (ndim == 3 ? 4 : 0), label_bytes + 4 * planes2 + 4, two.n_cut,
                     "feature transform", chunks)))
    return rc;

  // the intermediate distances: dist_out, or bit-cast in the last axis's index plane, which phase 2
  // reads them from before it writes that plane
  float* mid = dist_out ? dist_out : reinterpret_cast<float*>(idx_out[last]);
  rc = run_phase(dc, device, two.p1, label_bytes, planes1, [&](const ChunkSlots& slots, PipelineSteps& steps) {
    steps.item = "phase-1 chunk";
    steps.upload = [&](int k, int slot, cudaStream_t s) {
      return upload_box(slots.labels[slot], two.slab(labels, k, label_bytes), device, s);
    };
    steps.passes = [&](int k, int slot, cudaStream_t s) {
      const int64_t c = two.p1.size(k);
      const void* lab = slots.labels[slot];
      return with_label_width(label_bytes, [&](auto b) {
        int r = launch_first_sites<b>(lab, slots.plane(slot, 0), slots.plane<int>(slot, ndim == 3 ? 2 : 1),
                                      two.plane / sx * c, sx, wx, border, kernel_flags(flags, true, false), dc, s);
        if (r || ndim == 2) return r;
        r = launch_later_sites<b>(lab, slots.plane(slot, 0), slots.plane(slot, 1), slots.plane<int>(slot, 3),
                                  geom_for_axis(1, sx, sy, c), wy, border, border, kernel_flags(flags, false, false),
                                  transform_arith(t.w, t.n, 1), dc, s);
        return r ? r : launch_slice_sites<b>(lab, slots.plane<int>(slot, 2), slots.plane<int>(slot, 3), sx, sy, c,
                                             zero_bg, slots.plane<int32_t>(slot, 0), dc, s);
      });
    };
    steps.download = [&](int k, int slot, cudaStream_t s) {
      int r = download_box(two.slab(mid, k, 4), slots.plane(slot, ndim == 3 ? 1 : 0), device, s);
      if (!r) r = download_box(two.slab(idx_out[0], k, 4), slots.plane(slot, ndim == 3 ? 0 : 1), device, s);
      if (!r && ndim == 3) r = download_box(two.slab(idx_out[1], k, 4), slots.plane(slot, 3), device, s);
      return r;
    };
  });
  if (rc) return rc;
  return run_phase(dc, device, two.p2, label_bytes, planes2, [&](const ChunkSlots& slots, PipelineSteps& steps) {
    steps.item = "phase-2 chunk";
    steps.upload_writes_results = true;            // volume 0 goes up and comes back down as x
    steps.upload = [&](int k, int slot, cudaStream_t s) {
      int r = upload_box(slots.labels[slot], two.lines(labels, k, label_bytes), device, s);
      if (!r) r = upload_box(slots.plane(slot, 0), two.lines(mid, k, 4), device, s);
      for (int a = 0; !r && a < ndim - 1; ++a)
        r = upload_box(slots.plane(slot, 2 + a), two.lines(idx_out[a], k, 4), device, s);
      return r;
    };
    steps.passes = [&](int k, int slot, cudaStream_t s) {
      const int64_t c = two.p2.size(k);
      const edtb200::LineGeom g = ndim == 3 ? geom_for_axis(2, sx, c, sz) : geom_for_axis(1, c, sy, 1);
      const edtb200::SiteBox sb{ndim, ndim == 3 ? sx : c, two.unit * c, two.n_last, two.p2.start(k)};
      const void* lab = slots.labels[slot];
      return with_label_width(label_bytes, [&](auto b) {
        const int r = launch_later_sites<b>(lab, slots.plane(slot, 0), slots.plane(slot, 1),
                                            slots.plane<int>(slot, codes), g, t.w[last], border, border,
                                            kernel_flags(flags, false, true), transform_arith(t.w, t.n, last), dc, s);
        return r ? r : launch_compose_sites<b>(lab, slots.plane<int>(slot, codes), slots.plane<int32_t>(slot, 2),
                                               ndim == 3 ? slots.plane<int32_t>(slot, 3) : nullptr, sb, zero_bg,
                                               slots.plane<int32_t>(slot, 0),
                                               ndim == 3 ? slots.plane<int32_t>(slot, 5) : nullptr, dc, s);
      });
    };
    steps.download = [&](int k, int slot, cudaStream_t s) {
      int r = dist_out ? download_box(two.lines(dist_out, k, 4), slots.plane(slot, 1), device, s) : 0;
      if (!r) r = download_box(two.lines(idx_out[0], k, 4), slots.plane(slot, 0), device, s);
      if (!r && ndim == 3) r = download_box(two.lines(idx_out[1], k, 4), slots.plane(slot, 5), device, s);
      if (!r) r = download_box(two.lines(idx_out[last], k, 4), slots.plane(slot, codes), device, s);
      return r;
    };
  });
}

// Slot bytes of one group of edtb200_transform_stack on host buffers (include/edt_b200.h).
constexpr size_t kStackGroupBytes = size_t(512) << 20;

int edtb200_transform_stack(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                            int64_t count, float wx, float wy, float wz, int black_border, int flags, float* out,
                            int device, size_t device_bytes, int64_t* groups, void* stream_v) {
  if (groups) *groups = 0;
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  const int64_t vol = sx * sy * sz;
  if (vol == 0 || count == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  const bool in_dev = flags & EDTB200_LABELS_ON_DEVICE, out_dev = flags & EDTB200_OUT_ON_DEVICE;
  if (in_dev != out_dev)
    return fail(EDTB200_EINVAL, "edtb200_transform_stack takes labels and out both on the device or both on the host");
  const size_t vol_lab = (size_t)vol * (size_t)label_bytes, vol_out = (size_t)vol * sizeof(float);
  if (!in_dev && (rc = check_overlap({{labels, vol_lab * (size_t)count, "labels", false},
                                      {out, vol_out * (size_t)count, "out", true}})))
    return rc;

  StreamingCall call;
  if ((rc = call.open(device))) return rc;
  DeviceCache& dc = *call.dc;
  const int border = black_border != 0;
  if (in_dev) {                                  // asynchronous on the caller's stream, no lock
    rc = run_passes(labels, label_bytes, ndim, sx, sy, sz, wx, wy, wz, border, flags, out, dc,
                    static_cast<cudaStream_t>(stream_v), count);
    if (!rc && groups) *groups = 1;
    return rc;
  }

  // Host buffers: groups of whole volumes through two device slots, planned as a phase of
  // edtb200_transform_chunked whose slices are volumes.
  if ((rc = call.lock(device_bytes))) return rc;
  const Transform t{label_bytes, ndim, flags, border, {wx, wy, wz}, {sx, sy, sz}};
  bool long_any = false;                         // a later pass takes the long-line kernel: its scratch
  for (int k = 1; k < ndim; ++k)
    long_any = long_any || later_pass_is_long(geom_for_axis(k, sx, sy, sz), transform_arith(t.w, t.n, k),
                                              dc.max_smem_optin);
  // A group holds at most kStackGroupBytes of slot, so that a large stack runs as several groups whose
  // uploads and downloads overlap each other's passes, as edtb200_transform_batch's volumes do.
  const size_t voxel_bytes = label_bytes + 4 + (long_any ? 8 : 0);
  const int64_t most = std::max<int64_t>(1, (int64_t)(kStackGroupBytes / ((size_t)vol * voxel_bytes)));
  const PhasePlan p = call.plan(count, vol, voxel_bytes, most);
  if (p.count == 0)
    return fail(EDTB200_ENOMEM, "a device budget of %zu bytes cannot hold one group of volumes: the stack needs at "
                                "least %zu bytes", call.budget, p.need);
  if (p.count > 0x7fffffffLL) return fail(EDTB200_ELIMIT, "too many groups of volumes");
  const char* lab_host = static_cast<const char*>(labels);
  rc = run_phase(dc, device, p, label_bytes, 1, [&](const ChunkSlots& slots, PipelineSteps& steps) {
    steps.item = "group";
    steps.upload = [&](int k, int slot, cudaStream_t s) {
      return upload(slots.labels[slot], lab_host + (size_t)p.start(k) * vol_lab, (size_t)p.size(k) * vol_lab,
                    device, s);
    };
    steps.passes = [&](int k, int slot, cudaStream_t s) {
      return run_passes(slots.labels[slot], label_bytes, ndim, sx, sy, sz, wx, wy, wz, border, flags,
                        slots.plane(slot, 0), dc, s, p.size(k));
    };
    steps.download = [&](int k, int slot, cudaStream_t s) {
      return download(out + p.start(k) * vol, slots.plane(slot, 0), (size_t)p.size(k) * vol_out, device, s);
    };
  });
  if (rc) return rc;
  if (groups) *groups = p.count;
  return 0;
}

}  // extern "C"

namespace {

// max_distance: null for the unbounded feature transform, else the bounded one's (count 1), checked
// after the pointers.
int feature_transform_any(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                          int64_t count, float wx, float wy, float wz, int black_border, int flags, float* dist_out,
                          int32_t* const* idx_out, int device, void* stream_v, const double* max_distance) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  const int64_t vol = sx * sy * sz;
  if (vol == 0 || count == 0) return 0;
  if (!labels || !idx_out) return fail(EDTB200_EINVAL, "null pointer");
  for (int k = 0; k < ndim; ++k)
    if (!idx_out[k]) return fail(EDTB200_EINVAL, "null index plane %d", k);
  if (max_distance && !(*max_distance >= 0.0))
    return fail(EDTB200_EINVAL, "max_distance must be zero or more (got %g)", *max_distance);
  BoundedPlan plan;
  const BoundedPlan* bp = nullptr;
  if (max_distance && !std::isinf(*max_distance)) {
    const float w[3] = {wx, wy, wz};
    plan = bounded_plan(ndim, w, *max_distance, /*sites=*/true);
    bp = &plan;
  }
  const int64_t total = vol * count;

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  // host index planes are staged through one scratch; a distance volume and an index plane are 4 bytes
  // per voxel
  const size_t vol_bytes = (size_t)total * sizeof(float);
  const void* d_labels = nullptr;
  float* d_dist = nullptr;
  if ((rc = io.in_labels(labels, (size_t)total * (size_t)label_bytes, &d_labels)) ||
      (dist_out && (rc = io.out_dist(dist_out, vol_bytes, &d_dist))))
    return rc;
  Scratch planes;
  if (!io.out_dev && (rc = planes.take(*io.dc, (size_t)ndim * vol_bytes, io.stream, "the index planes"))) return rc;
  int32_t* d_idx[3] = {nullptr, nullptr, nullptr};
  for (int k = 0; k < ndim; ++k)
    d_idx[k] = io.out(idx_out[k], vol_bytes, io.out_dev ? nullptr : planes.get<int32_t>() + (size_t)k * total);
  rc = run_feature_passes(d_labels, label_bytes, ndim, sx, sy, sz, wx, wy, wz, black_border != 0, flags, d_dist,
                          d_idx, *io.dc, io.stream, count, bp);
  return rc ? rc : io.finish();
}

}  // namespace

extern "C" {

int edtb200_feature_transform_stack(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy,
                                    int64_t sz, int64_t count, float wx, float wy, float wz, int black_border,
                                    int flags, float* dist_out, int32_t* const* idx_out, int device, void* stream_v) {
  return feature_transform_any(labels, label_bytes, ndim, sx, sy, sz, count, wx, wy, wz, black_border, flags,
                               dist_out, idx_out, device, stream_v, nullptr);
}

int edtb200_feature_transform_bounded(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy,
                                      int64_t sz, float wx, float wy, float wz, int black_border, int flags,
                                      float* dist_out, int32_t* const* idx_out, int device, void* stream_v,
                                      double max_distance) {
  return feature_transform_any(labels, label_bytes, ndim, sx, sy, sz, 1, wx, wy, wz, black_border, flags, dist_out,
                               idx_out, device, stream_v, &max_distance);
}

int edtb200_transform_bounded(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                              float wx, float wy, float wz, int black_border, int flags, float* out, int device,
                              void* stream_v, double max_distance) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  const int64_t total = sx * sy * sz;
  if (total == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  if (!(max_distance >= 0.0)) return fail(EDTB200_EINVAL, "max_distance must be zero or more (got %g)", max_distance);
  if (std::isinf(max_distance))
    return edtb200_transform(labels, label_bytes, ndim, sx, sy, sz, wx, wy, wz, black_border, flags, out, device,
                             stream_v);
  const float w[3] = {wx, wy, wz};
  const BoundedPlan bp = bounded_plan(ndim, w, max_distance, /*sites=*/false);

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const void* d_labels = nullptr;
  float* d_out = nullptr;
  if ((rc = io.in_labels(labels, (size_t)total * (size_t)label_bytes, &d_labels)) ||
      (rc = io.out_dist(out, (size_t)total * sizeof(float), &d_out)))
    return rc;
  rc = run_bounded_passes(d_labels, label_bytes, ndim, sx, sy, sz, wx, wy, wz, black_border != 0, flags, d_out, bp,
                          *io.dc, io.stream);
  return rc ? rc : io.finish();
}

int edtb200_bounded_plan(int ndim, int64_t sx, int64_t sy, int64_t sz, float wx, float wy, float wz,
                         double max_distance, int64_t radius[3], int windowed[3]) {
  int rc = check_dims(1, ndim, sx, sy, sz);
  if (rc) return rc;
  if (!(max_distance >= 0.0)) return fail(EDTB200_EINVAL, "max_distance must be zero or more (got %g)", max_distance);
  if (!radius || !windowed) return fail(EDTB200_EINVAL, "null pointer");
  const float w[3] = {wx, wy, wz};
  const BoundedPlan bp = bounded_plan(ndim, w, max_distance, false), sp = bounded_plan(ndim, w, max_distance, true);
  for (int k = 0; k < 3; ++k) {
    radius[k] = k < ndim ? bp.radius[k] : 0;
    windowed[k] = k < ndim ? (bp.windowed[k] ? 1 : 0) | (sp.windowed[k] ? 2 : 0) : 0;
  }
  return 0;
}

int edtb200_morphology(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                       int64_t count, float wx, float wy, float wz, int op, double radius, int black_border, int flags,
                       void* out, int device, void* stream_v) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (op < EDTB200_ERODE || op > EDTB200_CLOSE) return fail(EDTB200_EINVAL, "op must be EDTB200_ERODE, _DILATE, _OPEN or _CLOSE (got %d)", op);
  if (!(radius >= 0.0) || std::isinf(radius))
    return fail(EDTB200_EINVAL, "radius must be finite and zero or more (got %g)", radius);
  const int known = EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE | EDTB200_LABELS_FLOAT;
  if (flags & ~known)
    return fail(EDTB200_EINVAL, "edtb200_morphology takes only the residency flags and EDTB200_LABELS_FLOAT (got %d)",
                flags);
  if ((rc = check_float_labels(flags, label_bytes))) return rc;
  const bool as_float = flags & EDTB200_LABELS_FLOAT;
  const int64_t vol = sx * sy * sz;
  if ((rc = check_stack(vol, count, 1))) return rc;
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  const float w[3] = {wx, wy, wz};
  const BoundedPlan bp = bounded_plan(ndim, w, radius, /*sites=*/false);
  const bool mask_out = op == EDTB200_DILATE || op == EDTB200_CLOSE;
  const int border = black_border != 0;

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const cudaStream_t s = io.stream;
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes;
  const void* d_labels = nullptr;
  void* d_out = nullptr;
  if ((rc = io.in_labels(labels, lab_bytes, &d_labels)) ||
      (rc = io.out_dist(out, (size_t)total * (mask_out ? 1 : (size_t)label_bytes), &d_out)))
    return rc;
  // scratch: the distances, the first step's mask (opening, closing) and the folded float labels
  const bool two = op == EDTB200_OPEN || op == EDTB200_CLOSE;
  const char* what = "the morphology's scratch";
  Scratch dist, mask, folded;
  if ((rc = dist.take(*io.dc, sizeof(float) * (size_t)total, s, what)) ||
      (two && (rc = mask.take(*io.dc, (size_t)total, s, what))) ||
      (as_float && (rc = folded.take(*io.dc, lab_bytes, s, what))))
    return rc;
  const void* runs = d_labels;                   // the labels the transforms compare
  if (as_float) {
    if ((rc = launch_fold_float_labels(d_labels, label_bytes, folded.get(), total, *io.dc, s))) return rc;
    runs = folded.get();
  }
  // select tables, bit (2 nz + near): erode keeps nz & !near (4), dilate sets nz | near (2, 4, 8), open's
  // mask is 0 on the erosion E and 1 elsewhere (the complement of 4), open keeps nz & near (8)
  constexpr int kErode = 0x4, kDilate = 0xE, kNotEroded = 0xB, kNear = 0x8;
  auto step = [&](const void* lab, int lab_w, int bord, int fl, const edtb200::MorphSelect& sel) {
    return run_bounded_passes(lab, lab_w, ndim, sx, sy, sz, wx, wy, wz, bord, fl, dist.get<float>(), bp, *io.dc, s,
                              count, &sel);
  };
  uint8_t* m = mask.get<uint8_t>();
  switch (op) {
    case EDTB200_ERODE:
      rc = step(runs, label_bytes, border, 0, {d_labels, d_out, label_bytes, kErode, false, as_float});
      break;
    case EDTB200_DILATE:
      rc = step(runs, label_bytes, 0, EDTB200_SIGNED, {d_labels, d_out, label_bytes, kDilate, true, as_float});
      break;
    case EDTB200_OPEN:        // the erosion E as a mask, then d^2(p, E) = edtsq of that mask
      rc = step(runs, label_bytes, border, 0, {d_labels, m, label_bytes, kNotEroded, true, as_float});
      if (!rc) rc = step(m, 1, 0, 0, {d_labels, d_out, label_bytes, kNear, false, as_float});
      break;
    default:                  // EDTB200_CLOSE: the dilation D as a mask, then D eroded as a two-label volume
      rc = step(runs, label_bytes, 0, EDTB200_SIGNED, {d_labels, m, label_bytes, kDilate, true, as_float});
      if (!rc) rc = step(m, 1, border, 0, {m, d_out, 1, kErode, true, false});
      break;
  }
  return rc ? rc : io.finish();
}

int edtb200_local_thickness(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                            int64_t count, float wx, float wy, float wz, int black_border, int flags,
                            const double* sizes, int nsizes, float* out, double* sizes_out, int device,
                            void* stream_v) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  const float w[3] = {wx, wy, wz};
  if ((rc = check_weights(ndim, w))) return rc;
  if (nsizes < 1 || nsizes > EDTB200_THICKNESS_MAX_SIZES)
    return fail(EDTB200_EINVAL, "nsizes must be 1 to %d (got %d)", EDTB200_THICKNESS_MAX_SIZES, nsizes);
  if (sizes)
    for (int i = 0; i < nsizes; ++i)
      if (!(sizes[i] >= 0.0) || std::isinf(sizes[i]))
        return fail(EDTB200_EINVAL, "sizes[%d] must be finite and zero or more (got %g)", i, sizes[i]);
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE | EDTB200_LABELS_FLOAT))
    return fail(EDTB200_EINVAL,
                "edtb200_local_thickness takes only the residency flags and EDTB200_LABELS_FLOAT (got %d)", flags);
  if ((rc = check_float_labels(flags, label_bytes))) return rc;
  const bool as_float = flags & EDTB200_LABELS_FLOAT;
  const int64_t vol = sx * sy * sz;
  if ((rc = check_stack(vol, count, 1))) return rc;
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, out_bytes = sizeof(float) * (size_t)total;
  const size_t levels_bytes = sizeof(double) * (size_t)count * (size_t)nsizes;
  if (same_side(flags) && overlaps(labels, lab_bytes, out, out_bytes)) return fail(EDTB200_EINVAL, "out overlaps labels");
  if (sizes_out && overlaps(sizes_out, levels_bytes, out, out_bytes))
    return fail(EDTB200_EINVAL, "sizes_out overlaps out");
  if (sizes_out && same_side(flags) && overlaps(sizes_out, levels_bytes, labels, lab_bytes))
    return fail(EDTB200_EINVAL, "sizes_out overlaps labels");
  // the levels a caller gave, descending; a repeated level is run once
  std::vector<double> given;
  if (sizes) given.assign(sizes, sizes + nsizes);
  std::sort(given.begin(), given.end(), [](double a, double b) { return a > b; });

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const cudaStream_t s = io.stream;
  const void* d_labels = nullptr;
  float* d_out = nullptr;
  if ((rc = io.in_labels(labels, lab_bytes, &d_labels)) || (rc = io.out_dist(out, out_bytes, &d_out))) return rc;
  // scratch: D2, the mask and the mask's distances (9 bytes per voxel), the folded float labels, and with
  // default levels their table (r staged for a host sizes_out, or kept in scratch without one), cuts and tops
  Scratch d2, mask, d2r, folded, table, staged;
  const char* what = "local thickness's scratch";
  const bool by_default = !sizes;
  double* d_levels = nullptr;
  if ((rc = d2.take(*io.dc, sizeof(float) * (size_t)total, s, what)) ||
      (rc = mask.take(*io.dc, (size_t)total, s, what)) ||
      (rc = d2r.take(*io.dc, sizeof(float) * (size_t)total, s, what)) ||
      (as_float && (rc = folded.take(*io.dc, lab_bytes, s, what))))
    return rc;
  if (sizes_out && (by_default || io.out_dev) &&
      (rc = io.out_staged(sizes_out, levels_bytes, staged, "the levels", &d_levels)))
    return rc;
  const size_t cuts_bytes = sizeof(float) * (size_t)count * (size_t)nsizes;
  if (by_default &&
      (rc = table.take(*io.dc, (d_levels ? 0 : levels_bytes) + cuts_bytes + sizeof(unsigned) * (size_t)count, s, what)))
    return rc;
  const void* runs = d_labels;                   // the labels the edtsq compares
  if (as_float) {
    if ((rc = launch_fold_float_labels(d_labels, label_bytes, folded.get(), total, *io.dc, s))) return rc;
    runs = folded.get();
  }
  StepTimer timer(s);
  timer.stamp();
  rc = run_passes(runs, label_bytes, ndim, sx, sy, sz, wx, wy, wz, black_border != 0, 0, d2.get<float>(), *io.dc, s,
                  count);
  float* cuts = nullptr;
  if (!rc && by_default) {
    char* base = table.get<char>();
    if (!d_levels) { d_levels = reinterpret_cast<double*>(base); base += levels_bytes; }
    cuts = reinterpret_cast<float*>(base);
    unsigned* top = reinterpret_cast<unsigned*>(base + cuts_bytes);
    const double h = (double)*std::min_element(w, w + ndim);
    rc = launch_thickness_top(d_labels, label_bytes, as_float, d2.get<float>(), vol, count, top, *io.dc, s);
    if (!rc) rc = launch_thickness_levels(top, count, nsizes, h, d_levels, cuts, *io.dc, s);
  }
  timer.stamp();
  // per level: the seeds, the edtsq of the mask, the store
  bool first = true;
  for (int i = 0; !rc && i < nsizes; ++i) {
    edtb200::ThicknessLevel level{nullptr, nullptr, 0, 0.0, 0.0f};
    if (by_default) {
      level = {d_levels + i, cuts + i, nsizes, 0.0, 0.0f};
    } else {
      level.r0 = given[i];
      level.b0 = edtb200::cut_bound(given[i]);
      if (sizes_out && !io.out_dev)
        for (int64_t v = 0; v < count; ++v) sizes_out[v * nsizes + i] = given[i];
      else if (sizes_out && (rc = launch_thickness_fill(d_levels, count, nsizes, i, given[i], *io.dc, s)))
        break;
      if (i > 0 && given[i] == given[i - 1]) continue;
    }
    rc = launch_thickness_seed(d2.get<float>(), vol, count, level, mask.get<uint8_t>(), *io.dc, s);
    if (!rc)
      rc = run_passes(mask.get(), 1, ndim, sx, sy, sz, wx, wy, wz, 0, 0, d2r.get<float>(), *io.dc, s, count);
    if (!rc)
      rc = launch_thickness_store(d_labels, label_bytes, as_float, d2r.get<float>(), vol, count, level, first, d_out,
                                  *io.dc, s);
    first = false;
  }
  timer.stamp();
  if (!rc && timer.synchronize())
    fprintf(stderr, "[edt_b200] local_thickness %lldx%lldx%lld x%lld L=%d  edtsq and levels %.3f ms  %d levels %.3f ms\n",
            (long long)sx, (long long)sy, (long long)sz, (long long)count, label_bytes, timer.ms(0, 1), nsizes,
            timer.ms(1, 2));
  return rc ? rc : io.finish();
}

// edtb200_parabolic, and with sites edtb200_parabolic_sites.
static int parabolic_any(const float* f, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count, float wx,
                         float wy, float wz, int op, int flags, float* out, bool sites, int32_t* idx, int device,
                         void* stream_v) {
  const char* name = sites ? "edtb200_parabolic_sites" : "edtb200_parabolic";
  int rc = check_dims(4, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (op != EDTB200_PARABOLIC_ERODE && op != EDTB200_PARABOLIC_DILATE)
    return fail(EDTB200_EINVAL, "op must be EDTB200_PARABOLIC_ERODE or _DILATE (got %d)", op);
  const float w[3] = {wx, wy, wz};
  if ((rc = check_weights(ndim, w))) return rc;
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "%s takes only the residency flags (got %d)", name, flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = check_stack(vol, count, 1))) return rc;
  // with sites, (i-j)^2 must be exact in double on the brute-force lines
  if (sites && (sx > kParabolicSitesN || sy > kParabolicSitesN || sz > kParabolicSitesN))
    return fail(EDTB200_ELIMIT, "%s takes lines of at most 2^26 samples", name);
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!f || !out || (sites && !idx)) return fail(EDTB200_EINVAL, "null pointer");
  const size_t bytes = sizeof(float) * (size_t)total, idx_bytes = (size_t)ndim * bytes;
  if (same_side(flags) && f != out && overlaps(f, bytes, out, bytes))
    return fail(EDTB200_EINVAL, "out overlaps f without being f");
  if (idx && overlaps(idx, idx_bytes, out, bytes)) return fail(EDTB200_EINVAL, "idx overlaps out");
  if (idx && same_side(flags) && overlaps(idx, idx_bytes, f, bytes)) return fail(EDTB200_EINVAL, "idx overlaps f");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const cudaStream_t s = io.stream;
  const float* d_f = nullptr;
  float* d_out = nullptr;
  if ((rc = io.in_labels(f, bytes, &d_f)) || (rc = io.out_dist(out, bytes, &d_out))) return rc;
  // sites: the index planes (staged for a host idx), and the code planes of every pass but the last,
  // whose codes go straight into its own index plane (the resolver reads them only at their own voxel)
  Scratch staged, planes;
  int32_t* d_idx = nullptr;
  int* codes[3] = {nullptr, nullptr, nullptr};
  if (idx) {
    if ((rc = io.out_staged(idx, idx_bytes, staged, "the index planes", &d_idx)) ||
        (ndim > 1 && (rc = planes.take(*io.dc, (size_t)(ndim - 1) * bytes, s, "the site code planes"))))
      return rc;
    for (int k = 0; k < ndim; ++k) codes[k] = (k == ndim - 1 ? d_idx : planes.get<int32_t>()) + (size_t)k * total;
  }
  StepTimer timer(s);
  timer.stamp();
  int kernel[3];
  rc = parabolic_passes(d_f, d_out, ndim, sx, sy, sz, count, w, op == EDTB200_PARABOLIC_DILATE, codes, kernel, timer,
                        *io.dc, s);
  if (!rc && idx) {
    int32_t* const planes_out[3] = {d_idx, d_idx + total, d_idx + 2 * (size_t)total};
    rc = launch_resolve_sites<1>(nullptr, codes, ndim, sx, sy, sz, count, false, planes_out, *io.dc, s);
  }
  if (!rc && timer.synchronize()) {
    static const char* names[4] = {"tile", "long", "brute", "copy"};
    fprintf(stderr, "[edt_b200] parabolic %s %lldx%lldx%lld x%lld  x %.3f ms (%s)  y %.3f ms (%s)  z %.3f ms (%s)\n",
            op == EDTB200_PARABOLIC_DILATE ? "dilate" : "erode", (long long)sx, (long long)sy, (long long)sz,
            (long long)count, timer.ms(0, 1), names[kernel[0] < 0 ? 0 : kernel[0]], timer.ms(1, 2),
            kernel[1] < 0 ? "-" : names[kernel[1]], timer.ms(2, 3), kernel[2] < 0 ? "-" : names[kernel[2]]);
  }
  return rc ? rc : io.finish();
}

int edtb200_parabolic(const float* f, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count, float wx,
                      float wy, float wz, int op, int flags, float* out, int device, void* stream_v) {
  return parabolic_any(f, ndim, sx, sy, sz, count, wx, wy, wz, op, flags, out, false, nullptr, device, stream_v);
}

int edtb200_parabolic_sites(const float* f, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count, float wx,
                            float wy, float wz, int op, int flags, float* out, int32_t* idx, int device,
                            void* stream_v) {
  return parabolic_any(f, ndim, sx, sy, sz, count, wx, wy, wz, op, flags, out, true, idx, device, stream_v);
}

int edtb200_medial_axis(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                        int64_t count, float wx, float wy, float wz, int black_border, int flags, uint8_t* medial_out,
                        float* dist_out, int device, void* stream_v) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  const float w[3] = {wx, wy, wz};
  if ((rc = check_weights(ndim, w))) return rc;
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE | EDTB200_LABELS_FLOAT))
    return fail(EDTB200_EINVAL, "edtb200_medial_axis takes only the residency flags and EDTB200_LABELS_FLOAT (got %d)",
                flags);
  if ((rc = check_float_labels(flags, label_bytes))) return rc;
  const bool as_float = flags & EDTB200_LABELS_FLOAT;
  const int64_t vol = sx * sy * sz;
  if ((rc = check_stack(vol, count, 1))) return rc;
  // the sites' limit: beyond it (i-j)^2 is not exact in double on the brute-force lines
  if (sx > kParabolicSitesN || sy > kParabolicSitesN || sz > kParabolicSitesN)
    return fail(EDTB200_ELIMIT, "edtb200_medial_axis takes lines of at most 2^26 samples");
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !medial_out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, dist_bytes = sizeof(float) * (size_t)total;
  if (same_side(flags) && overlaps(labels, lab_bytes, medial_out, (size_t)total))
    return fail(EDTB200_EINVAL, "medial_out overlaps labels");
  if (dist_out && same_side(flags) && overlaps(labels, lab_bytes, dist_out, dist_bytes))
    return fail(EDTB200_EINVAL, "dist_out overlaps labels");
  if (dist_out && overlaps(medial_out, (size_t)total, dist_out, dist_bytes))
    return fail(EDTB200_EINVAL, "dist_out overlaps medial_out");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const cudaStream_t s = io.stream;
  // host buffers are staged whole: the labels and distances through this device's cached buffers, the
  // mask through scratch
  const void* d_labels = nullptr;
  uint8_t* d_medial = nullptr;
  float* d_dist = nullptr;
  Scratch staged, values, planes;
  if ((rc = io.in_labels(labels, lab_bytes, &d_labels)) ||
      (rc = io.out_staged(medial_out, (size_t)total, staged, "the medial mask", &d_medial)) ||
      (dist_out && (rc = io.out_dist(dist_out, dist_bytes, &d_dist))))
    return rc;
  // scratch: one value volume (D^2 without distances, the dilation's values with them) and the code
  // planes, which hold the folded float labels until the edtsq has read them
  const size_t plane_bytes = std::max(dist_bytes * (size_t)ndim, as_float ? lab_bytes : 0);
  if ((rc = values.take(*io.dc, dist_bytes, s, "the medial axis's scratch")) ||
      (rc = planes.take(*io.dc, plane_bytes, s, "the medial axis's scratch")))
    return rc;
  const void* runs = d_labels;                   // the labels the edtsq compares
  if (as_float) {
    if ((rc = launch_fold_float_labels(d_labels, label_bytes, planes.get(), total, *io.dc, s))) return rc;
    runs = planes.get();
  }
  float* d2 = d_dist ? d_dist : values.get<float>();
  int* codes[3] = {nullptr, nullptr, nullptr};
  for (int k = 0; k < ndim; ++k) codes[k] = planes.get<int>() + (size_t)k * total;

  // steps: the edtsq, a pass per axis, the mark
  StepTimer timer(s);
  timer.stamp();
  rc = run_passes(runs, label_bytes, ndim, sx, sy, sz, wx, wy, wz, black_border != 0, 0, d2, *io.dc, s, count);
  timer.stamp();
  int kernel[3];
  // with distances the first pass writes the value scratch
  if (!rc)
    rc = parabolic_passes(d2, values.get<float>(), ndim, sx, sy, sz, count, w, /*dilate=*/true, codes, kernel, timer,
                          *io.dc, s);
  if (!rc && cudaMemsetAsync(d_medial, 0, (size_t)total, s) != cudaSuccess)
    rc = fail(EDTB200_ECUDA, "cudaMemsetAsync of the medial mask failed");
  if (!rc)
    rc = launch_medial_mark(d_labels, label_bytes, codes, ndim, sx, sy, sz, count, as_float, d_medial, d_dist, *io.dc,
                            s);
  timer.stamp();
  if (!rc && timer.synchronize()) {
    static const char* names[4] = {"tile", "long", "brute", "copy"};
    fprintf(stderr, "[edt_b200] medial_axis %lldx%lldx%lld x%lld L=%d  edtsq %.3f ms  x %.3f ms (%s)  y %.3f ms (%s)  "
                    "z %.3f ms (%s)  mark %.3f ms\n",
            (long long)sx, (long long)sy, (long long)sz, (long long)count, label_bytes, timer.ms(0, 1), timer.ms(1, 2),
            names[kernel[0] < 0 ? 0 : kernel[0]], ndim > 1 ? timer.ms(2, 3) : 0.0f,
            kernel[1] < 0 ? "-" : names[kernel[1]], ndim > 2 ? timer.ms(3, 4) : 0.0f,
            kernel[2] < 0 ? "-" : names[kernel[2]], timer.ms(ndim + 1, ndim + 2));
  }
  return rc ? rc : io.finish();
}

int edtb200_skeletonize(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                        int64_t count, float wx, float wy, float wz, int black_border, int flags,
                        uint8_t* skeleton_out, float* dist_out, int device, void* stream_v) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (ndim < 2) return fail(EDTB200_EINVAL, "edtb200_skeletonize takes 2-D and 3-D volumes (got ndim %d)", ndim);
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  const float w[3] = {wx, wy, wz};
  if ((rc = check_weights(ndim, w))) return rc;
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_skeletonize takes only the residency flags (got %d)", flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = check_stack(vol, count, 1))) return rc;
  // one list segment holds the voxels of one subfield: 4-byte entries
  const int64_t cap = count * ((sx + 1) / 2) * ((sy + 1) / 2) * ((sz + 1) / 2);
  if (cap >= ((int64_t)1 << 32))
    return fail(EDTB200_ELIMIT, "edtb200_skeletonize takes stacks of fewer than 2^32 voxels per subfield");
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !skeleton_out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, dist_bytes = sizeof(float) * (size_t)total;
  if (same_side(flags) && overlaps(labels, lab_bytes, skeleton_out, (size_t)total))
    return fail(EDTB200_EINVAL, "skeleton_out overlaps labels");
  if (dist_out && same_side(flags) && overlaps(labels, lab_bytes, dist_out, dist_bytes))
    return fail(EDTB200_EINVAL, "dist_out overlaps labels");
  if (dist_out && overlaps(skeleton_out, (size_t)total, dist_out, dist_bytes))
    return fail(EDTB200_EINVAL, "dist_out overlaps skeleton_out");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const cudaStream_t s = io.stream;
  // host buffers are staged whole: the labels and distances through this device's cached buffers, the
  // skeleton through scratch
  const void* d_labels = nullptr;
  uint8_t* d_skel = nullptr;
  float* d_dist = nullptr;
  Scratch staged, values, list, control;
  if ((rc = io.in_labels(labels, lab_bytes, &d_labels)) ||
      (rc = io.out_staged(skeleton_out, (size_t)total, staged, "the skeleton", &d_skel)) ||
      (dist_out && (rc = io.out_dist(dist_out, dist_bytes, &d_dist))))
    return rc;
  // scratch: the edtsq when no distances are wanted, then -- once the edtsq has returned its own scratch to
  // the pool -- the two list buffers of one segment per subfield and the control block (the state plane is
  // the skeleton's buffer)
  if (!d_dist && (rc = values.take(*io.dc, dist_bytes, s, "the skeleton's edtsq"))) return rc;
  SkeletonScratch sk;
  sk.segments = ndim == 3 ? 8 : 4;
  sk.cap = (uint32_t)cap;
  const size_t list_bytes = 2 * (size_t)sk.segments * (size_t)cap * sizeof(uint32_t);
  float* d2 = d_dist ? d_dist : values.get<float>();
  float h = wx;
  for (int k = 1; k < ndim; ++k) h = std::min(h, w[k]);

  // steps: the edtsq, the thinning
  StepTimer timer(s);
  timer.stamp();
  rc = run_passes(d_labels, label_bytes, ndim, sx, sy, sz, wx, wy, wz, black_border != 0, 0, d2, *io.dc, s, count);
  timer.stamp();
  if (!rc) rc = list.take(*io.dc, list_bytes, s, "the skeleton's lists");
  if (!rc) rc = control.take(*io.dc, skeleton_control_bytes(), s, "the skeleton's lists");
  sk.list = list.get<uint32_t>();
  sk.control = control.get();
  if (!rc)
    rc = launch_skeleton_thin(d_labels, label_bytes, ndim, sx, sy, sz, count, h, d2, sk, d_skel, d_dist, *io.dc, s);
  timer.stamp();
  if (!rc && timer.synchronize()) {
    unsigned long long n[3] = {0, 0, 0};
    skeleton_stats(sk.control, n);
    fprintf(stderr, "[edt_b200] skeletonize %lldx%lldx%lld x%lld L=%d  edtsq %.3f ms  thin %.3f ms  rounds %llu  "
                    "cycles %llu  steps %llu  scratch %zu bytes\n",
            (long long)sx, (long long)sy, (long long)sz, (long long)count, label_bytes, timer.ms(0, 1), timer.ms(1, 2),
            n[0], n[1], n[2], (d_dist ? 0 : dist_bytes) + list_bytes + skeleton_control_bytes());
  }
  return rc ? rc : io.finish();
}

int edtb200_geodesic(const void* labels, int label_bytes, const void* seeds, int seed_bytes, int ndim, int64_t sx,
                     int64_t sy, int64_t sz, int64_t count, float wx, float wy, float wz, int flags, float* dist_out,
                     int32_t* const* idx_out, int device, void* stream_v) {
  if (!(label_bytes == 1 || label_bytes == 2 || label_bytes == 4 || label_bytes == 8))
    return fail(EDTB200_EINVAL, "label_bytes must be 1, 2, 4 or 8 (got %d)", label_bytes);
  if (!(seed_bytes == 1 || seed_bytes == 2 || seed_bytes == 4 || seed_bytes == 8))
    return fail(EDTB200_EINVAL, "seed_bytes must be 1, 2, 4 or 8 (got %d)", seed_bytes);
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  const float w[3] = {wx, wy, wz};
  if ((rc = check_weights(ndim, w))) return rc;
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_geodesic takes only the residency flags (got %d)", flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = check_stack(vol, count, 1))) return rc;
  // the worklists hold 4-byte tile numbers
  const int64_t ntiles = geodesic_tiles(ndim, sx, sy, sz, count);
  if (ntiles >= ((int64_t)1 << 32)) return fail(EDTB200_ELIMIT, "edtb200_geodesic takes stacks of fewer than 2^32 tiles");
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !seeds || !dist_out) return fail(EDTB200_EINVAL, "null pointer");
  if (idx_out)
    for (int k = 0; k < ndim; ++k)
      if (!idx_out[k]) return fail(EDTB200_EINVAL, "null index plane %d", k);
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, seed_size = (size_t)total * (size_t)seed_bytes;
  const size_t dist_bytes = sizeof(float) * (size_t)total, plane_bytes = sizeof(int32_t) * (size_t)total;
  // outputs against the inputs (on the same side) and against each other
  const void* outs[4] = {dist_out, idx_out ? idx_out[0] : nullptr, idx_out && ndim > 1 ? idx_out[1] : nullptr,
                         idx_out && ndim > 2 ? idx_out[2] : nullptr};
  const size_t out_bytes[4] = {dist_bytes, plane_bytes, plane_bytes, plane_bytes};
  static const char* names[4] = {"dist_out", "index plane 0", "index plane 1", "index plane 2"};
  for (int i = 0; i < 4; ++i) {
    if (!outs[i]) continue;
    if (same_side(flags) && overlaps(labels, lab_bytes, outs[i], out_bytes[i]))
      return fail(EDTB200_EINVAL, "%s overlaps labels", names[i]);
    if (same_side(flags) && overlaps(seeds, seed_size, outs[i], out_bytes[i]))
      return fail(EDTB200_EINVAL, "%s overlaps seeds", names[i]);
    for (int j = 0; j < i; ++j)
      if (outs[j] && overlaps(outs[j], out_bytes[j], outs[i], out_bytes[i]))
        return fail(EDTB200_EINVAL, "%s overlaps %s", names[i], names[j]);
  }

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const cudaStream_t s = io.stream;
  // host buffers are staged whole: the labels and distances through this device's cached buffers, the
  // seeds and index planes through scratch
  const void* d_labels = nullptr;
  const void* d_seeds = nullptr;
  float* d_dist = nullptr;
  int32_t* d_planes[3] = {nullptr, nullptr, nullptr};
  Scratch seed_stage, plane_stage[3], values, indices, tiles;
  if ((rc = io.in_labels(labels, lab_bytes, &d_labels)) || (rc = io.out_dist(dist_out, dist_bytes, &d_dist)))
    return rc;
  if (!io.in_dev && (rc = seed_stage.take(*io.dc, seed_size, s, "the staged seeds"))) return rc;
  if ((rc = io.in(seeds, seed_size, seed_stage.get(), &d_seeds))) return rc;
  for (int k = 0; idx_out && k < ndim; ++k)
    if ((rc = io.out_staged(idx_out[k], plane_bytes, plane_stage[k], "the index planes", &d_planes[k]))) return rc;
  // scratch: D, S with indices, one flag and two list entries per tile, and the two control blocks
  GeodesicScratch g;
  g.ntiles = ntiles;
  const size_t tile_bytes = 3 * sizeof(uint32_t) * (size_t)ntiles, d_bytes = sizeof(double) * (size_t)total;
  const size_t s_bytes = idx_out ? sizeof(unsigned long long) * (size_t)total : 0;
  if ((rc = values.take(*io.dc, d_bytes, s, "the geodesic distances")) ||
      (idx_out && (rc = indices.take(*io.dc, s_bytes, s, "the geodesic seed indices"))) ||
      (rc = tiles.take(*io.dc, tile_bytes + geodesic_control_bytes(), s, "the geodesic worklists")))
    return rc;
  g.d = values.get<double>();
  g.s = indices.get<unsigned long long>();
  // the control blocks first: they hold 8-byte counters, and 3 * ntiles words may end off an 8-byte boundary
  g.control = tiles.get();
  g.flag = reinterpret_cast<uint32_t*>(tiles.get<char>() + geodesic_control_bytes());
  g.list = g.flag + ntiles;
  // the step lengths: each weight promoted to double, the squares summed in the order x, y, z, sqrt
  double step[8] = {0.0};
  for (int m = 1; m < 8; ++m) {
    double sum = 0.0;
    for (int k = 0; k < 3; ++k)
      if (m >> k & 1) sum += (double)w[k] * (double)w[k];
    step[m] = std::sqrt(sum);
  }

  // steps: the distances, the indices, the store
  StepTimer timer(s);
  timer.stamp();
  rc = launch_geodesic_phase(d_labels, label_bytes, d_seeds, seed_bytes, ndim, sx, sy, sz, count, step, g, false,
                             *io.dc, s);
  timer.stamp();
  if (!rc && idx_out)
    rc = launch_geodesic_phase(d_labels, label_bytes, d_seeds, seed_bytes, ndim, sx, sy, sz, count, step, g, true,
                               *io.dc, s);
  timer.stamp();
  if (!rc) rc = launch_geodesic_store(ndim, sx, sy, sz, count, g, d_dist, idx_out ? d_planes : nullptr, *io.dc, s);
  timer.stamp();
  if (!rc && timer.synchronize()) {
    unsigned long long n[4] = {0, 0, 0, 0};
    geodesic_stats(g.control, n);
    fprintf(stderr, "[edt_b200] geodesic %lldx%lldx%lld x%lld L=%d  distances %.3f ms (rounds %llu, tile visits %llu)  "
                    "indices %.3f ms (rounds %llu, tile visits %llu)  store %.3f ms  tiles %lld  scratch %zu bytes\n",
            (long long)sx, (long long)sy, (long long)sz, (long long)count, label_bytes, timer.ms(0, 1), n[0], n[1],
            timer.ms(1, 2), n[2], n[3], timer.ms(2, 3), (long long)ntiles,
            d_bytes + s_bytes + tile_bytes + geodesic_control_bytes());
  }
  return rc ? rc : io.finish();
}

int edtb200_watershed(const void* labels, int label_bytes, const void* markers, int marker_bytes, const float* image,
                      int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count, int connectivity, int flags,
                      void* out, float* level_out, int device, void* stream_v) {
  if (!(label_bytes == 0 || label_bytes == 1 || label_bytes == 2 || label_bytes == 4 || label_bytes == 8))
    return fail(EDTB200_EINVAL, "label_bytes must be 0 (no labels), 1, 2, 4 or 8 (got %d)", label_bytes);
  if (!(marker_bytes == 1 || marker_bytes == 2 || marker_bytes == 4 || marker_bytes == 8))
    return fail(EDTB200_EINVAL, "marker_bytes must be 1, 2, 4 or 8 (got %d)", marker_bytes);
  int rc = check_dims(label_bytes ? label_bytes : 1, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (connectivity < 1 || connectivity > ndim)
    return fail(EDTB200_EINVAL, "connectivity must be 1 to ndim (%d) (got %d)", ndim, connectivity);
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_watershed takes only the residency flags (got %d)", flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = check_stack(vol, count, 1))) return rc;
  // the worklists hold 4-byte tile numbers
  const int64_t ntiles = geodesic_tiles(ndim, sx, sy, sz, count);
  if (ntiles >= ((int64_t)1 << 32)) return fail(EDTB200_ELIMIT, "edtb200_watershed takes stacks of fewer than 2^32 tiles");
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if ((label_bytes && !labels) || !markers || !image || !out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, marker_size = (size_t)total * (size_t)marker_bytes;
  const size_t image_bytes = sizeof(float) * (size_t)total, out_bytes = marker_size;
  // outputs against the inputs (on the same side) and against each other
  const void* outs[2] = {out, level_out};
  const size_t outs_bytes[2] = {out_bytes, image_bytes};
  static const char* names[2] = {"out", "level_out"};
  for (int i = 0; i < 2; ++i) {
    if (!outs[i]) continue;
    if (same_side(flags) && label_bytes && overlaps(labels, lab_bytes, outs[i], outs_bytes[i]))
      return fail(EDTB200_EINVAL, "%s overlaps labels", names[i]);
    if (same_side(flags) && overlaps(markers, marker_size, outs[i], outs_bytes[i]))
      return fail(EDTB200_EINVAL, "%s overlaps markers", names[i]);
    if (same_side(flags) && overlaps(image, image_bytes, outs[i], outs_bytes[i]))
      return fail(EDTB200_EINVAL, "%s overlaps image", names[i]);
  }
  if (level_out && overlaps(out, out_bytes, level_out, image_bytes))
    return fail(EDTB200_EINVAL, "level_out overlaps out");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const cudaStream_t s = io.stream;
  // host buffers are staged whole: the labels and levels through this device's cached buffers, the markers,
  // the image and the result through scratch
  const void* d_labels = nullptr;
  const void* d_markers = nullptr;
  const float* d_image = nullptr;
  void* d_out = nullptr;
  float* d_level = nullptr;
  Scratch marker_stage, image_stage, out_stage, values, wsheds, tiles;
  if (label_bytes && (rc = io.in_labels(labels, lab_bytes, &d_labels))) return rc;
  if (level_out && (rc = io.out_dist(level_out, image_bytes, &d_level))) return rc;
  if (!io.in_dev && ((rc = marker_stage.take(*io.dc, marker_size, s, "the staged markers")) ||
                     (rc = image_stage.take(*io.dc, image_bytes, s, "the staged image"))))
    return rc;
  if ((rc = io.in(markers, marker_size, marker_stage.get(), &d_markers)) ||
      (rc = io.in(image, image_bytes, image_stage.get(), &d_image)) ||
      (rc = io.out_staged(out, out_bytes, out_stage, "the watershed labels", &d_out)))
    return rc;
  // scratch: L, W, one flag and two list entries per tile, and the two control blocks
  WatershedScratch g;
  g.ntiles = ntiles;
  const size_t tile_bytes = 3 * sizeof(uint32_t) * (size_t)ntiles, l_bytes = sizeof(float) * (size_t)total;
  const size_t w_bytes = (marker_bytes == 8 ? 8 : 4) * (size_t)total;
  if ((rc = values.take(*io.dc, l_bytes, s, "the watershed levels")) ||
      (rc = wsheds.take(*io.dc, w_bytes, s, "the watershed markers")) ||
      (rc = tiles.take(*io.dc, tile_bytes + watershed_control_bytes(), s, "the watershed worklists")))
    return rc;
  g.level = values.get<float>();
  g.w = wsheds.get();
  // the control blocks first: they hold 8-byte counters, and 3 * ntiles words may end off an 8-byte boundary
  g.control = tiles.get();
  g.flag = reinterpret_cast<uint32_t*>(tiles.get<char>() + watershed_control_bytes());
  g.list = g.flag + ntiles;

  // steps: the levels, the labels, the store
  StepTimer timer(s);
  timer.stamp();
  rc = launch_watershed_phase(d_labels, label_bytes, d_markers, marker_bytes, d_image, ndim, sx, sy, sz, count,
                              connectivity, g, false, *io.dc, s);
  timer.stamp();
  if (!rc)
    rc = launch_watershed_phase(d_labels, label_bytes, d_markers, marker_bytes, d_image, ndim, sx, sy, sz, count,
                                connectivity, g, true, *io.dc, s);
  timer.stamp();
  if (!rc) rc = launch_watershed_store(ndim, sx, sy, sz, count, marker_bytes, g, d_out, d_level, *io.dc, s);
  timer.stamp();
  if (!rc && timer.synchronize()) {
    unsigned long long n[4] = {0, 0, 0, 0};
    watershed_stats(g.control, n);
    fprintf(stderr, "[edt_b200] watershed %lldx%lldx%lld x%lld L=%d M=%d c=%d  levels %.3f ms (rounds %llu, tile visits "
                    "%llu)  labels %.3f ms (rounds %llu, tile visits %llu)  store %.3f ms  tiles %lld  scratch %zu bytes\n",
            (long long)sx, (long long)sy, (long long)sz, (long long)count, label_bytes, marker_bytes, connectivity,
            timer.ms(0, 1), n[0], n[1], timer.ms(1, 2), n[2], n[3], timer.ms(2, 3), (long long)ntiles,
            l_bytes + w_bytes + tile_bytes + watershed_control_bytes());
  }
  return rc ? rc : io.finish();
}

// The checks edtb200_connected_components and edtb200_extended_maxima share after their own, in their
// documented order: out_bytes, the stack's size, the volume's size (parents are 4-byte indices within a volume)
// and the output width against it.
static int components_checks(const char* name, int64_t vol, int64_t count, int out_bytes) {
  if (out_bytes != 4 && out_bytes != 8) return fail(EDTB200_EINVAL, "out_bytes must be 4 or 8 (got %d)", out_bytes);
  if (const int rc = check_stack(vol, count, 1)) return rc;
  if (vol >= ((int64_t)1 << 32)) return fail(EDTB200_ELIMIT, "%s takes volumes of fewer than 2^32 voxels", name);
  if (out_bytes == 4 && vol >= ((int64_t)1 << 31))
    return fail(EDTB200_EINVAL, "out_bytes 4 needs volumes of fewer than 2^31 voxels (got %lld)", (long long)vol);
  return 0;
}

// The union-find passes and the numbering of one call, device buffers in place; h > 0 first reconstructs -R
// from the image.  Prints the phases with EDT_B200_VERBOSE.
static int components_run(const char* name, ComponentsJob j, const float* image, double h, void* out, HostIO& io) {
  const cudaStream_t s = io.stream;
  const int64_t total = j.sx * j.sy * j.sz * j.count;
  const size_t temp_bytes = components_temp_bytes(total, j.count, j.out_bytes);
  const size_t p_bytes = sizeof(uint32_t) * (size_t)total;
  Scratch parents, temp, values, tiles;
  int rc;
  if ((rc = parents.take(*io.dc, p_bytes, s, "the component parents")) ||
      (rc = temp.take(*io.dc, temp_bytes, s, "the component numbering")))
    return rc;
  j.parent = parents.get<uint32_t>();
  size_t extra = 0;
  WatershedScratch g;
  if (image && h > 0.0) {
    // -R and -f, one flag and two list entries per tile, and the control blocks
    g.ntiles = geodesic_tiles(j.ndim, j.sx, j.sy, j.sz, j.count);
    const size_t tile_bytes = 3 * sizeof(uint32_t) * (size_t)g.ntiles;
    extra = 2 * sizeof(float) * (size_t)total + tile_bytes + watershed_control_bytes();
    if ((rc = values.take(*io.dc, 2 * sizeof(float) * (size_t)total, s, "the reconstruction")) ||
        (rc = tiles.take(*io.dc, tile_bytes + watershed_control_bytes(), s, "the reconstruction worklists")))
      return rc;
    g.level = values.get<float>();
    g.control = tiles.get();
    g.flag = reinterpret_cast<uint32_t*>(tiles.get<char>() + watershed_control_bytes());
    g.list = g.flag + g.ntiles;
  }
  // steps: [the reconstruction,] the union, the flatten (and mark), the numbering
  StepTimer timer(s);
  timer.stamp();
  rc = 0;
  if (g.level) {
    rc = launch_hmax_phase(j.labels, j.label_bytes, image, h, g.level + total, j.ndim, j.sx, j.sy, j.sz, j.count,
                           j.connectivity, g, *io.dc, s);
    j.value = g.level;
    j.negated = true;
    timer.stamp();
  } else {
    j.value = image;
  }
  if (!rc) rc = launch_components_union(j, *io.dc, s);
  timer.stamp();
  if (!rc) rc = launch_components_flatten(j, out, *io.dc, s);
  timer.stamp();
  if (!rc) rc = launch_components_number(j, out, temp.get(), temp_bytes, *io.dc, s);
  timer.stamp();
  if (!rc && timer.synchronize()) {
    const int k = g.level ? 1 : 0;
    unsigned long long n[4] = {0, 0, 0, 0};
    if (g.level) watershed_stats(g.control, n);
    fprintf(stderr, "[edt_b200] %s %lldx%lldx%lld x%lld L=%d c=%d  reconstruction %.3f ms (rounds %llu, tile visits "
                    "%llu)  union %.3f ms  flatten%s %.3f ms  numbering %.3f ms  scratch %zu bytes\n",
            name, (long long)j.sx, (long long)j.sy, (long long)j.sz, (long long)j.count, j.label_bytes, j.connectivity,
            k ? timer.ms(0, 1) : 0.0f, n[0], n[1], timer.ms(k, k + 1), image ? " and mark" : "",
            timer.ms(k + 1, k + 2), timer.ms(k + 2, k + 3), p_bytes + temp_bytes + extra);
  }
  return rc;
}

int edtb200_connected_components(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                                 int64_t count, int connectivity, int flags, void* out, int out_bytes, int device,
                                 void* stream_v) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (connectivity < 1 || connectivity > ndim)
    return fail(EDTB200_EINVAL, "connectivity must be 1 to ndim (%d) (got %d)", ndim, connectivity);
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_connected_components takes only the residency flags (got %d)", flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = components_checks("edtb200_connected_components", vol, count, out_bytes))) return rc;
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, res_bytes = (size_t)total * (size_t)out_bytes;
  if (same_side(flags) && overlaps(labels, lab_bytes, out, res_bytes)) return fail(EDTB200_EINVAL, "out overlaps labels");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const void* d_labels = nullptr;
  void* d_out = nullptr;
  Scratch out_stage;
  if ((rc = io.in_labels(labels, lab_bytes, &d_labels)) ||
      (rc = io.out_staged(out, res_bytes, out_stage, "the components", &d_out)))
    return rc;
  ComponentsJob j;
  j.labels = d_labels;
  j.label_bytes = label_bytes;
  j.ndim = ndim; j.sx = sx; j.sy = sy; j.sz = sz; j.count = count;
  j.connectivity = connectivity;
  j.out_bytes = out_bytes;
  rc = components_run("connected_components", j, nullptr, 0.0, d_out, io);
  return rc ? rc : io.finish();
}

int edtb200_extended_maxima(const void* labels, int label_bytes, const float* image, int ndim, int64_t sx, int64_t sy,
                            int64_t sz, int64_t count, double h, int connectivity, int flags, void* out, int out_bytes,
                            int device, void* stream_v) {
  if (!(label_bytes == 0 || label_bytes == 1 || label_bytes == 2 || label_bytes == 4 || label_bytes == 8))
    return fail(EDTB200_EINVAL, "label_bytes must be 0 (no labels), 1, 2, 4 or 8 (got %d)", label_bytes);
  int rc = check_dims(label_bytes ? label_bytes : 1, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (!(std::isfinite(h) && h >= 0.0)) return fail(EDTB200_EINVAL, "h must be finite and >= 0 (got %g)", h);
  if (connectivity < 1 || connectivity > ndim)
    return fail(EDTB200_EINVAL, "connectivity must be 1 to ndim (%d) (got %d)", ndim, connectivity);
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_extended_maxima takes only the residency flags (got %d)", flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = components_checks("edtb200_extended_maxima", vol, count, out_bytes))) return rc;
  // the reconstruction's worklists hold 4-byte tile numbers
  if (h > 0.0 && geodesic_tiles(ndim, sx, sy, sz, count) >= ((int64_t)1 << 32))
    return fail(EDTB200_ELIMIT, "edtb200_extended_maxima with h > 0 takes stacks of fewer than 2^32 tiles");
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if ((label_bytes && !labels) || !image || !out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, image_bytes = sizeof(float) * (size_t)total;
  const size_t res_bytes = (size_t)total * (size_t)out_bytes;
  if (same_side(flags) && label_bytes && overlaps(labels, lab_bytes, out, res_bytes))
    return fail(EDTB200_EINVAL, "out overlaps labels");
  if (same_side(flags) && overlaps(image, image_bytes, out, res_bytes)) return fail(EDTB200_EINVAL, "out overlaps image");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  // host buffers are staged whole: the labels through this device's cached buffer, the image and the result
  // through scratch
  const void* d_labels = nullptr;
  const float* d_image = nullptr;
  void* d_out = nullptr;
  Scratch image_stage, out_stage;
  if (label_bytes && (rc = io.in_labels(labels, lab_bytes, &d_labels))) return rc;
  if (!io.in_dev && (rc = image_stage.take(*io.dc, image_bytes, io.stream, "the staged image"))) return rc;
  if ((rc = io.in(image, image_bytes, image_stage.get(), &d_image)) ||
      (rc = io.out_staged(out, res_bytes, out_stage, "the maxima", &d_out)))
    return rc;
  ComponentsJob j;
  j.labels = d_labels;
  j.label_bytes = label_bytes;
  j.ndim = ndim; j.sx = sx; j.sy = sy; j.sz = sz; j.count = count;
  j.connectivity = connectivity;
  j.out_bytes = out_bytes;
  rc = components_run("extended_maxima", j, d_image, h, d_out, io);
  return rc ? rc : io.finish();
}

// The checks edtb200_fill_holes and edtb200_dust share, in their documented order: label width, ndim and
// sizes, count >= 0, connectivity; after their own bound and flags they call holes_size_checks.
static int holes_checks(int label_bytes, int ndim, int64_t& sx, int64_t& sy, int64_t& sz, int64_t count,
                        int connectivity) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (connectivity < 1 || connectivity > ndim)
    return fail(EDTB200_EINVAL, "connectivity must be 1 to ndim (%d) (got %d)", ndim, connectivity);
  return 0;
}

// The stack's size and the volume's size (parents are 4-byte indices within a volume).
static int holes_size_checks(const char* name, int64_t vol, int64_t count) {
  if (const int rc = check_stack(vol, count, 1)) return rc;
  if (vol >= ((int64_t)1 << 32)) return fail(EDTB200_ELIMIT, "%s takes volumes of fewer than 2^32 voxels", name);
  return 0;
}

// The union, tally and apply passes of one call, device buffers in place.  Prints the phases with
// EDT_B200_VERBOSE.
static int holes_run(const char* name, HolesJob j, void* out, HostIO& io) {
  const cudaStream_t s = io.stream;
  const int64_t total = j.cc.sx * j.cc.sy * j.cc.sz * j.cc.count;
  const bool sized = !j.fill || j.bound != ~(uint64_t)0;
  const size_t p_bytes = sizeof(uint32_t) * (size_t)total, size_bytes = sized ? sizeof(uint32_t) * (size_t)total : 0;
  const size_t claim_bytes = j.fill ? (j.cc.label_bytes == 8 ? 8 : 4) * (size_t)total : 0;
  const size_t state_bytes = j.fill ? ((size_t)total + 3) & ~(size_t)3 : 0;
  Scratch parents, sizes, claims;
  int rc;
  if ((rc = parents.take(*io.dc, p_bytes, s, "the component parents")) ||
      (sized && (rc = sizes.take(*io.dc, size_bytes, s, "the component sizes"))) ||
      (j.fill && (rc = claims.take(*io.dc, claim_bytes + state_bytes, s, "the hole claims"))))
    return rc;
  j.cc.parent = parents.get<uint32_t>();
  j.size = sized ? sizes.get<uint32_t>() : nullptr;
  if (j.fill) {
    j.claim = claims.get();
    j.state = claims.get<uint8_t>() + claim_bytes;
  }
  // what the tally and apply accumulate into starts at zero
  if (sized) CUDA_TRY(cudaMemsetAsync(j.size, 0, size_bytes, s));
  if (j.fill) CUDA_TRY(cudaMemsetAsync(j.claim, 0, claim_bytes + state_bytes, s));
  if (j.counts) CUDA_TRY(cudaMemsetAsync(j.counts, 0, sizeof(unsigned long long) * (size_t)j.cc.count, s));
  // steps: the union, the tally, the apply
  StepTimer timer(s);
  timer.stamp();
  rc = launch_holes_union(j, *io.dc, s);
  timer.stamp();
  if (!rc) rc = launch_holes_tally(j, *io.dc, s);
  timer.stamp();
  if (!rc) rc = launch_holes_apply(j, out, *io.dc, s);
  timer.stamp();
  if (!rc && timer.synchronize())
    fprintf(stderr, "[edt_b200] %s %lldx%lldx%lld x%lld L=%d c=%d  union %.3f ms  tally %.3f ms  apply %.3f ms  "
                    "scratch %zu bytes\n",
            name, (long long)j.cc.sx, (long long)j.cc.sy, (long long)j.cc.sz, (long long)j.cc.count,
            j.cc.label_bytes, j.cc.connectivity, timer.ms(0, 1), timer.ms(1, 2), timer.ms(2, 3),
            p_bytes + size_bytes + claim_bytes + state_bytes);
  return rc;
}

int edtb200_fill_holes(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                       int64_t count, int connectivity, int64_t max_size, int flags, void* out, int64_t* fill_counts,
                       int device, void* stream_v) {
  int rc = holes_checks(label_bytes, ndim, sx, sy, sz, count, connectivity);
  if (rc) return rc;
  if (max_size < -1) return fail(EDTB200_EINVAL, "max_size must be -1 (none) or >= 0 (got %lld)", (long long)max_size);
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_fill_holes takes only the residency flags (got %d)", flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = holes_size_checks("edtb200_fill_holes", vol, count))) return rc;
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t res_bytes = (size_t)total * (size_t)label_bytes, counts_bytes = sizeof(int64_t) * (size_t)count;
  if (same_side(flags) && overlaps(labels, res_bytes, out, res_bytes)) return fail(EDTB200_EINVAL, "out overlaps labels");
  if (fill_counts && overlaps(fill_counts, counts_bytes, out, res_bytes))
    return fail(EDTB200_EINVAL, "fill_counts overlaps out");
  if (fill_counts && same_side(flags) && overlaps(fill_counts, counts_bytes, labels, res_bytes))
    return fail(EDTB200_EINVAL, "fill_counts overlaps labels");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const void* d_labels = nullptr;
  void* d_out = nullptr;
  int64_t* d_counts = nullptr;
  Scratch out_stage, counts_stage;
  if ((rc = io.in_labels(labels, res_bytes, &d_labels)) ||
      (rc = io.out_staged(out, res_bytes, out_stage, "the filled labels", &d_out)) ||
      (fill_counts && (rc = io.out_staged(fill_counts, counts_bytes, counts_stage, "the fill counts", &d_counts))))
    return rc;
  HolesJob j;
  j.cc.labels = d_labels;
  j.cc.label_bytes = label_bytes;
  j.cc.ndim = ndim; j.cc.sx = sx; j.cc.sy = sy; j.cc.sz = sz; j.cc.count = count;
  j.cc.connectivity = connectivity;
  j.fill = true;
  j.bound = max_size < 0 ? ~(uint64_t)0 : (uint64_t)max_size;
  j.counts = reinterpret_cast<unsigned long long*>(d_counts);
  rc = holes_run("fill_holes", j, d_out, io);
  return rc ? rc : io.finish();
}

int edtb200_dust(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz, int64_t count,
                 int connectivity, int64_t threshold, int invert, int flags, void* out, int device, void* stream_v) {
  int rc = holes_checks(label_bytes, ndim, sx, sy, sz, count, connectivity);
  if (rc) return rc;
  if (threshold < 0) return fail(EDTB200_EINVAL, "threshold must be >= 0 (got %lld)", (long long)threshold);
  if (invert != 0 && invert != 1) return fail(EDTB200_EINVAL, "invert must be 0 or 1 (got %d)", invert);
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_dust takes only the residency flags (got %d)", flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = holes_size_checks("edtb200_dust", vol, count))) return rc;
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t res_bytes = (size_t)total * (size_t)label_bytes;
  if (same_side(flags) && overlaps(labels, res_bytes, out, res_bytes)) return fail(EDTB200_EINVAL, "out overlaps labels");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const void* d_labels = nullptr;
  void* d_out = nullptr;
  Scratch out_stage;
  if ((rc = io.in_labels(labels, res_bytes, &d_labels)) ||
      (rc = io.out_staged(out, res_bytes, out_stage, "the dusted labels", &d_out)))
    return rc;
  HolesJob j;
  j.cc.labels = d_labels;
  j.cc.label_bytes = label_bytes;
  j.cc.ndim = ndim; j.cc.sx = sx; j.cc.sy = sy; j.cc.sz = sz; j.cc.count = count;
  j.cc.connectivity = connectivity;
  j.bound = (uint64_t)threshold;
  j.invert = invert != 0;
  rc = holes_run("dust", j, d_out, io);
  return rc ? rc : io.finish();
}

// The checks edtb200_nearest_labels and its plan share, in their documented order, up to max_distance.
static int nearest_checks(int label_bytes, int ndim, int64_t& sx, int64_t& sy, int64_t& sz, int64_t count,
                          const float w[3], int k, double max_distance) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if ((rc = check_weights(ndim, w))) return rc;
  if (k < 1 || k > 4) return fail(EDTB200_EINVAL, "k must be 1, 2, 3 or 4 (got %d)", k);
  if (!(max_distance >= 0.0) || std::isinf(max_distance))
    return fail(EDTB200_EINVAL, "max_distance must be finite and zero or more (got %g): the cost is O(R) per voxel "
                "per pass, so an unbounded call is not offered", max_distance);
  return 0;
}

int edtb200_nearest_labels_plan(int ndim, int64_t sx, int64_t sy, int64_t sz, float wx, float wy, float wz,
                                double max_distance, int k, int label_bytes, int64_t radius[3], int variant[3]) {
  const float w[3] = {wx, wy, wz};
  int rc = nearest_checks(label_bytes, ndim, sx, sy, sz, 1, w, k, max_distance);
  if (rc) return rc;
  if (!radius || !variant) return fail(EDTB200_EINVAL, "null pointer");
  const NearestPlan p = nearest_plan(ndim, w, max_distance, k, label_bytes);
  for (int a = 0; a < 3; ++a) {
    radius[a] = p.radius[a];
    variant[a] = p.variant[a];
  }
  return 0;
}

int edtb200_nearest_labels(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                           int64_t count, float wx, float wy, float wz, double max_distance, int k, int flags,
                           float* dist_out, void* label_out, int device, void* stream_v) {
  const float w[3] = {wx, wy, wz};
  int rc = nearest_checks(label_bytes, ndim, sx, sy, sz, count, w, k, max_distance);
  if (rc) return rc;
  const NearestPlan p = nearest_plan(ndim, w, max_distance, k, label_bytes);
  for (int a = 0; a < ndim; ++a)
    if (p.variant[a] < 0)
      return fail(EDTB200_ELIMIT, "the pass along axis %d needs a radius of %lld rows; the limit is %lld", a,
                  (long long)p.radius[a], (long long)kNearRadiusLimit);
  if (flags & ~(EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE | EDTB200_NEAREST_SQUARED))
    return fail(EDTB200_EINVAL, "edtb200_nearest_labels takes only the residency flags and EDTB200_NEAREST_SQUARED "
                "(got %d)", flags);
  const int64_t vol = sx * sy * sz;
  if ((rc = check_stack(vol, count, k))) return rc;
  const int64_t total = vol * count;
  if (total == 0) return 0;
  if (!labels || !dist_out || !label_out) return fail(EDTB200_EINVAL, "null pointer");
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes;
  const size_t dist_bytes = sizeof(float) * (size_t)total * (size_t)k, lout_bytes = lab_bytes * (size_t)k;
  if (overlaps(dist_out, dist_bytes, label_out, lout_bytes)) return fail(EDTB200_EINVAL, "dist_out overlaps label_out");
  if (same_side(flags) &&
      (overlaps(labels, lab_bytes, dist_out, dist_bytes) || overlaps(labels, lab_bytes, label_out, lout_bytes)))
    return fail(EDTB200_EINVAL, "an output overlaps labels");

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  const cudaStream_t s = io.stream;
  // host buffers are staged whole: the labels and distances through this device's cached buffers, the
  // output labels through scratch
  const void* d_labels = nullptr;
  float* d_dist = nullptr;
  void* d_lab = nullptr;
  Scratch staged, planes;
  if ((rc = io.in_labels(labels, lab_bytes, &d_labels)) || (rc = io.out_dist(dist_out, dist_bytes, &d_dist)) ||
      (rc = io.out_staged(label_out, lout_bytes, staged, "the output labels", &d_lab)))
    return rc;
  // the scratch set of the passes: k value and label planes (2-D and 3-D)
  float* sdist = nullptr;
  void* slab = nullptr;
  if (ndim > 1) {
    // the value planes from a 16-byte boundary after the label planes, which may end anywhere
    const size_t at = (lout_bytes + 15) & ~(size_t)15;
    if ((rc = planes.take(*io.dc, at + dist_bytes, s, "the passes' scratch planes"))) return rc;
    slab = planes.get();
    sdist = reinterpret_cast<float*>(planes.get<char>() + at);
  }
  rc = nearest_passes(d_labels, label_bytes, ndim, sx, sy, sz, count, w, p, k, !(flags & EDTB200_NEAREST_SQUARED),
                      d_dist, d_lab, sdist, slab, *io.dc, s);
  return rc ? rc : io.finish();
}

int edtb200_expand_gather(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                          int64_t count, const float* sqdist, const int32_t* const* idx, double limit_sq, int flags,
                          void* out, int device, void* stream_v) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (sx * sy * sz == 0 || count == 0) return 0;
  if (!labels || !sqdist || !idx) return fail(EDTB200_EINVAL, "null pointer");
  for (int k = 0; k < ndim; ++k)
    if (!idx[k]) return fail(EDTB200_EINVAL, "null index plane %d", k);
  if (!out) return fail(EDTB200_EINVAL, "null pointer");
  const int both = EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE;
  if ((flags & both) != both || (flags & ~(both | EDTB200_LABELS_FLOAT)))
    return fail(EDTB200_EINVAL, "edtb200_expand_gather works on device buffers only: flags must be "
                                "EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE, optionally with EDTB200_LABELS_FLOAT "
                                "(got %d)", flags);
  if ((rc = check_float_labels(flags, label_bytes))) return rc;
  const bool as_float = flags & EDTB200_LABELS_FLOAT;

  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  if ((rc = probe(device, &dc))) return rc;
  const int32_t* planes[3] = {idx[0], ndim >= 2 ? idx[1] : nullptr, ndim >= 3 ? idx[2] : nullptr};
  return with_label_width(label_bytes, [&](auto b) {        // asynchronous on the caller's stream, no lock
    return launch_expand_gather<b>(labels, sqdist, planes, ndim, sx, sy, sz, count, limit_sq, as_float, out, *dc,
                                   static_cast<cudaStream_t>(stream_v));
  });
}

}  // extern "C"

namespace {

constexpr int64_t kSurfaceGroupVoxels = int64_t(1) << 31;   // mask voxels of one group of surface slots

// The checks edtb200_surface_count and edtb200_surface_distances share before their pointers: the
// geometry, count, nkeys and the host keys (non-zero, strictly ascending as unsigned integers of
// label_bytes).  *empty: nothing to do (no voxel, no volume or no key).
int check_surface(int label_bytes, int ndim, int64_t& sx, int64_t& sy, int64_t& sz, int64_t count, const void* keys,
                  int64_t nkeys, bool* empty) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (count < 0) return fail(EDTB200_EINVAL, "negative count");
  if (nkeys < 0) return fail(EDTB200_EINVAL, "negative nkeys");
  if (nkeys > 0 && !keys) return fail(EDTB200_EINVAL, "null pointer (keys)");
  uint64_t prev = 0;
  for (int64_t k = 0; k < nkeys; ++k) {
    uint64_t key = 0;
    memcpy(&key, static_cast<const char*>(keys) + k * label_bytes, (size_t)label_bytes);   // little-endian
    if (key == 0) return fail(EDTB200_EINVAL, "key %lld is 0 (background)", (long long)k);
    if (k > 0 && key <= prev) return fail(EDTB200_EINVAL, "keys must be strictly ascending (key %lld)", (long long)k);
    prev = key;
  }
  if (nkeys > 0 && count > ((int64_t)1 << 60) / nkeys) return fail(EDTB200_ELIMIT, "too many (volume, key) pairs");
  *empty = sx * sy * sz == 0 || count == 0 || nkeys == 0;
  return 0;
}

int check_surface_flags(int flags, const char* name) {
  const int both = EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE;
  if (flags != both)
    return fail(EDTB200_EINVAL, "%s works on device buffers only: flags must be EDTB200_LABELS_ON_DEVICE | "
                                "EDTB200_OUT_ON_DEVICE (got %d)", name, flags);
  return 0;
}

// The keys on the device, for the kernels' search.
int upload_keys(Scratch& dev, const void* keys, int64_t nkeys, int label_bytes, DeviceCache& dc, cudaStream_t s) {
  const size_t bytes = (size_t)nkeys * (size_t)label_bytes;
  if (const int rc = dev.take(dc, bytes, s, "the keys")) return rc;
  CUDA_TRY(cudaMemcpyAsync(dev.get(), keys, bytes, cudaMemcpyHostToDevice, s));
  return 0;
}

}  // namespace

extern "C" {

int edtb200_surface_count(const void* a, const void* b, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                          int64_t count, const void* keys, int64_t nkeys, int flags, int64_t* counts, int device,
                          void* stream_v) {
  bool empty = false;
  int rc = check_surface(label_bytes, ndim, sx, sy, sz, count, keys, nkeys, &empty);
  if (rc || empty) return rc;
  if (!a || !b || !counts) return fail(EDTB200_EINVAL, "null pointer");
  if ((rc = check_surface_flags(flags, "edtb200_surface_count"))) return rc;

  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  if ((rc = probe(device, &dc))) return rc;
  const cudaStream_t s = static_cast<cudaStream_t>(stream_v);
  const int64_t slots = count * nkeys * 2;
  Scratch dev_keys;
  if ((rc = upload_keys(dev_keys, keys, nkeys, label_bytes, *dc, s))) return rc;
  CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(int64_t) * (size_t)slots, s));
  const edtb200::SurfaceSlots g{ndim, sx, sy, sz, sx * sy * sz, nkeys, 0, slots, 0, count};
  return with_label_width(label_bytes, [&](auto w) {
    return launch_surface<w>(a, b, dev_keys.get(), g, nullptr, nullptr, reinterpret_cast<unsigned long long*>(counts),
                             nullptr, *dc, s);
  });
}

int edtb200_surface_distances(const void* a, const void* b, int label_bytes, int ndim, int64_t sx, int64_t sy,
                              int64_t sz, int64_t count, float wx, float wy, float wz, const void* keys, int64_t nkeys,
                              int flags, const int64_t* offsets, float* values, int device, size_t device_bytes,
                              int64_t* groups, void* stream_v) {
  if (groups) *groups = 0;
  bool empty = false;
  int rc = check_surface(label_bytes, ndim, sx, sy, sz, count, keys, nkeys, &empty);
  if (rc || empty) return rc;
  if (!a || !b || !offsets || !values) return fail(EDTB200_EINVAL, "null pointer");
  if ((rc = check_surface_flags(flags, "edtb200_surface_distances"))) return rc;

  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  if ((rc = probe(device, &dc))) return rc;
  const cudaStream_t s = static_cast<cudaStream_t>(stream_v);
  const int64_t vol = sx * sy * sz, slots = count * nkeys * 2;
  // A slot costs its mask, its distances and, where a later pass takes the long-line kernel, that
  // kernel's two scratch volumes: the stack planner's rule (edtb200_transform_stack).
  const float w[3] = {wx, wy, wz};
  const int64_t n[3] = {sx, sy, sz};
  bool long_any = false;
  for (int k = 1; k < ndim; ++k)
    long_any = long_any || later_pass_is_long(geom_for_axis(k, sx, sy, sz), transform_arith(w, n, k), dc->max_smem_optin);
  const size_t slot_bytes = (size_t)vol * (1 + 4 + (long_any ? 8 : 0));
  size_t budget = device_bytes;
  if (budget == 0) {
    size_t free_bytes = 0, total_bytes = 0;
    CUDA_TRY(cudaMemGetInfo(&free_bytes, &total_bytes));
    budget = free_bytes > EDTB200_CHUNK_RESERVE ? free_bytes - EDTB200_CHUNK_RESERVE : 0;
  }
  const int64_t fit = std::min<int64_t>(slots, (int64_t)(budget / slot_bytes));
  if (fit == 0)
    return fail(EDTB200_ENOMEM, "a device budget of %zu bytes cannot hold one slot: the surface distances need at "
                                "least %zu bytes", budget, slot_bytes);
  // A group's masks hold at most kSurfaceGroupVoxels voxels (at least one slot), so that a call takes
  // no more memory than the transforms need to stream at full rate.
  const int64_t cap = std::max<int64_t>(1, kSurfaceGroupVoxels / vol);
  const int64_t fit_capped = std::min(fit, cap);
  const int64_t ngroups = (slots + fit_capped - 1) / fit_capped, most = (slots + ngroups - 1) / ngroups;

  Scratch dev_keys, cursor, buf;
  if ((rc = upload_keys(dev_keys, keys, nkeys, label_bytes, *dc, s))) return rc;
  // the distances of a group's slots, then their masks
  const size_t dist_bytes = ((size_t)most * (size_t)vol * 4 + 255) & ~size_t(255);
  if (cursor.alloc(*dc, sizeof(int64_t) * (size_t)slots, s) != cudaSuccess ||
      buf.alloc(*dc, dist_bytes + (size_t)most * (size_t)vol, s) != cudaSuccess) {
    cudaGetLastError();
    return fail(EDTB200_ENOMEM, "no device memory for a group of %lld slots", (long long)most);
  }
  auto* cur = cursor.get<unsigned long long>();
  float* dist = buf.get<float>();
  uint8_t* mask = buf.get<uint8_t>() + dist_bytes;
  CUDA_TRY(cudaMemcpyAsync(cur, offsets, sizeof(int64_t) * (size_t)slots, cudaMemcpyDeviceToDevice, s));
  for (int64_t grp = 0; grp < ngroups; ++grp) {
    const int64_t s0 = slots * grp / ngroups, s1 = slots * (grp + 1) / ngroups;
    const edtb200::SurfaceSlots g{ndim, sx, sy, sz, vol, nkeys, s0, s1, s0 / (2 * nkeys), (s1 - 1) / (2 * nkeys) + 1};
    CUDA_TRY(cudaMemsetAsync(mask, 1, (size_t)(s1 - s0) * (size_t)vol, s));
    rc = with_label_width(label_bytes, [&](auto lw) {
      return launch_surface<lw>(a, b, dev_keys.get(), g, mask, nullptr, nullptr, nullptr, *dc, s);
    });
    if (!rc) rc = run_passes(mask, 1, ndim, sx, sy, sz, wx, wy, wz, 0, EDTB200_SQRT, dist, *dc, s, s1 - s0);
    if (!rc) {
      rc = with_label_width(label_bytes, [&](auto lw) {
        return launch_surface<lw>(a, b, dev_keys.get(), g, nullptr, dist, cur + s0, values, *dc, s);
      });
    }
    if (rc) return rc;
  }
  if (groups) *groups = ngroups;
  return 0;
}

int edtb200_transform_voxel_graph(const void* labels, int label_bytes, const unsigned char* graph, int ndim,
                                  int64_t sx, int64_t sy, int64_t sz, float wx, float wy, float wz,
                                  int black_border, int flags, float* out, int device, void* stream_v) {
  using namespace edtb200;
  if (ndim != 2 && ndim != 3)
    return fail(EDTB200_EINVAL, "a voxel graph needs a 2-D or 3-D volume (got ndim %d)", ndim);
  if (flags & EDTB200_SIGNED)
    return fail(EDTB200_EINVAL, "EDTB200_SIGNED is not defined with a voxel graph: subtract two transforms");
  int rc = check_float_labels(flags, label_bytes);
  if (rc) return rc;
  if ((rc = check_dims(label_bytes, ndim, sx, sy, sz))) return rc;
  const int64_t total = sx * sy * sz;
  if (total == 0) return 0;
  if (!labels || !graph || !out) return fail(EDTB200_EINVAL, "null pointer");
  int64_t sx2 = 2 * sx, sy2 = 2 * sy, sz2 = ndim == 3 ? 2 * sz : 1;
  rc = check_dims(1, ndim, sx2, sy2, sz2);
  if (rc) return rc;
  const int64_t total2 = sx2 * sy2 * sz2;

  HostIO io;
  if ((rc = io.open(device, flags, stream_v))) return rc;
  DeviceCache* dc = io.dc;
  const cudaStream_t stream = io.stream;
  // stream-ordered scratch: the inputs when they come from the host, the doubled byte mask, the
  // doubled distance volume, and the result when it goes back to the host.  It is freed when the
  // call returns, after io.finish() has queued the download of the result.
  Scratch d_labels, d_graph, d_cells, d_doubled, d_result;
  if (!io.in_dev) {
    CUDA_TRY(d_labels.alloc(*dc, (size_t)total * label_bytes, stream));
    CUDA_TRY(d_graph.alloc(*dc, (size_t)total, stream));
  }
  const void* lab = nullptr;
  const uint8_t* gr = nullptr;
  if ((rc = io.in(labels, (size_t)total * label_bytes, d_labels.get(), &lab)) ||
      (rc = io.in(graph, (size_t)total, d_graph.get(), &gr)))
    return rc;
  CUDA_TRY(d_cells.alloc(*dc, (size_t)total2, stream));
  CUDA_TRY(d_doubled.alloc(*dc, (size_t)total2 * sizeof(float), stream));
  if (!io.out_dev) CUDA_TRY(d_result.alloc(*dc, (size_t)total * sizeof(float), stream));
  float* result = io.out(out, (size_t)total * sizeof(float), d_result.get<float>());

  const int threads = 256;
  const int blocks = (int)std::min<int64_t>((total + threads - 1) / threads, (int64_t)dc->sm_count * 32);
  const int border = black_border != 0, as_float = (flags & EDTB200_LABELS_FLOAT) ? 1 : 0;
  uint8_t* cells = d_cells.get<uint8_t>();
  rc = with_label_width(label_bytes, [&](auto b) {
    voxel_graph_expand_kernel<b><<<blocks, threads, 0, stream>>>(lab, gr, cells, sx, sy, sz, ndim, border, as_float,
                                                                 sy - 1, sz - 1);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
  if (rc) return rc;
  // half the anisotropy (vg:102-107, 199-204); the sqrt is taken by the gather instead
  rc = run_passes(cells, 1, ndim, sx2, sy2, sz2, wx / 2, wy / 2, wz / 2, border, 0, d_doubled.get<float>(), *dc,
                  stream);
  if (rc) return rc;
  voxel_graph_gather_kernel<<<blocks, threads, 0, stream>>>(d_doubled.get<const float>(), result, sx, sy, sz, 2,
                                                            4 * sx, 8 * sx * sy, (flags & EDTB200_SQRT) ? 1 : 0);
  CUDA_TRY(cudaGetLastError());
  return io.finish();
}

int edtb200_transform_voxel_graph_chunked(const void* labels, int label_bytes, const unsigned char* graph, int ndim,
                                          int64_t sx, int64_t sy, int64_t sz, float wx, float wy, float wz,
                                          int black_border, int flags, float* out, int device, size_t device_bytes,
                                          int64_t* chunks) {
  using namespace edtb200;
  if (chunks) chunks[0] = chunks[1] = 0;
  if (flags & (EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_transform_voxel_graph_chunked streams HOST buffers through the device; a "
                                "volume on the device fits it: use edtb200_transform_voxel_graph");
  if (ndim != 2 && ndim != 3)
    return fail(EDTB200_EINVAL, "a voxel graph needs a 2-D or 3-D volume (got ndim %d)", ndim);
  if (flags & EDTB200_SIGNED)
    return fail(EDTB200_EINVAL, "EDTB200_SIGNED is not defined with a voxel graph: subtract two transforms");
  int rc = check_float_labels(flags, label_bytes);
  if (rc) return rc;
  if ((rc = check_dims(label_bytes, ndim, sx, sy, sz))) return rc;
  const int64_t total = sx * sy * sz;
  if (total == 0) return 0;
  if (!labels || !graph || !out) return fail(EDTB200_EINVAL, "null pointer");
  int64_t sx2 = 2 * sx, sy2 = 2 * sy, sz2 = ndim == 3 ? 2 * sz : 1;
  if ((rc = check_dims(1, ndim, sx2, sy2, sz2))) return rc;
  const size_t lab_bytes = (size_t)total * (size_t)label_bytes, out_bytes = (size_t)total * sizeof(float);
  if ((rc = check_overlap({{labels, lab_bytes, "labels", false}, {graph, (size_t)total, "graph", false},
                           {out, out_bytes, "out", true}})))
    return rc;

  StreamingCall call;
  if ((rc = call.open(device)) || (rc = call.lock(device_bytes))) return rc;
  DeviceCache& dc = *call.dc;

  // The doubled grid's passes couple the cells of one line and the result samples even cells only,
  // so after the passes along the first axes each voxel carries two cells into the last pass: those
  // of its doubled line along the last axis at 2l and 2l + 1.
  //   phase 1  slabs across the last axis: the slab's doubled mask, the X pass (and in 3-D the Y
  //            pass over every doubled column), and the two cells per voxel come down: cell 2l into
  //            `out`, cell 2l + 1 into a host scratch;
  //   phase 2  boxes of whole lines along the last axis: both cells go up, are interleaved into the
  //            box's doubled lines beside their mask, the last pass runs, the even cells come down.
  // Every pass runs with the one-shot call's transform of the whole doubled grid.
  const int border = black_border != 0, as_float = (flags & EDTB200_LABELS_FLOAT) ? 1 : 0;
  const Transform t{1, ndim, 0, border, {wx / 2, wy / 2, wz / 2}, {sx2, sy2, sz2}};
  const int last = ndim - 1;
  TwoPhase two(ndim, sx, sy, sz);                          // cut in voxels, not doubled cells
  const int64_t plane = two.plane, n_last = two.n_last;
  const int cells = ndim == 3 ? 8 : 4;                     // doubled cells per voxel in phase 1
  const int64_t cap2 = std::max<int64_t>(1, (int64_t)((((int64_t)1 << 32) - 65) / (2 * two.line_vox)));
  const bool long1 = ndim == 3 && later_pass_is_long(geom_for_axis(1, sx2, sy2, sz2), transform_arith(t.w, t.n, 1),
                                                     dc.max_smem_optin);
  const int64_t c2 = std::min(two.n_cut, cap2);
  const LineGeom g2 = ndim == 3 ? geom_for_axis(2, sx, c2, sz2) : geom_for_axis(1, c2, sy2, 1);
  const bool long2 = later_pass_is_long(g2, transform_arith(t.w, t.n, last), dc.max_smem_optin);
  // Slot volumes (4 bytes per voxel each) beside the labels and the graph:
  //   phase 1  0 .. cells-1 the doubled distances; cells, cells+1 the two cells; then the doubled
  //            mask (cells / 4 volumes)
  //   phase 2  0, 1 the doubled lines; 2 cell 2l, then the result; 3 cell 2l + 1; 4 the lines' mask
  // and per launch of a later pass the long-line kernel's two scratch volumes of the doubled cells.
  const int planes1 = cells + 2 + cells / 4, planes2 = 5;
  if ((rc = two.plan(call, label_bytes + 1 + 4 * planes1 + (long1 ? 8 * cells : 0),
                     label_bytes + 1 + 4 * planes2 + (long2 ? 16 : 0), cap2, "voxel-graph transform", chunks)))
    return rc;
  std::unique_ptr<float, decltype(&free)> odd_cells(static_cast<float*>(malloc(out_bytes)), &free);
  if (!odd_cells)
    return fail(EDTB200_ENOMEM, "no host memory for the %zu-byte scratch of the odd cells between the phases",
                out_bytes);

  const int threads = 256;
  auto blocks = [&](int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + threads - 1) / threads,
                                                                                      (int64_t)dc.sm_count * 32)); };
  rc = run_phase(dc, device, two.p1, label_bytes + 1, planes1, [&](const ChunkSlots& slots, PipelineSteps& steps) {
    steps.item = "phase-1 chunk";
    steps.upload = [&](int k, int slot, cudaStream_t s) {
      const int r = upload_box(slots.labels[slot], two.slab(labels, k, label_bytes), device, s);
      return r ? r : upload_box(static_cast<char*>(slots.labels[slot]) + slots.vox * label_bytes, two.slab(graph, k, 1),
                                device, s);
    };
    steps.passes = [&](int k, int slot, cudaStream_t s) {
      const int64_t c = two.p1.size(k), z0 = two.p1.start(k);
      const int64_t cy = ndim == 3 ? sy : c, cz = ndim == 3 ? c : 1;              // the slab's extents
      const uint8_t* gr = reinterpret_cast<const uint8_t*>(slots.labels[slot]) + slots.vox * label_bytes;
      float* f = slots.plane(slot, 0);
      uint8_t* mask = slots.plane<uint8_t>(slot, cells + 2);
      int r = with_label_width(label_bytes, [&](auto b) {
        voxel_graph_expand_kernel<b><<<blocks(c * plane), threads, 0, s>>>(
            slots.labels[slot], gr, mask, sx, cy, cz, ndim, border, as_float,
            ndim == 3 ? sy - 1 : sy - 1 - z0, ndim == 3 ? sz - 1 - z0 : 0);
        CUDA_TRY(cudaGetLastError());
        return 0;
      });
      if (!r) r = x_pass(t, mask, f, 2 * cy * (ndim == 3 ? 2 * cz : 1), dc, s);
      if (!r && ndim == 3)                                  // behind our own X pass
        r = later_pass(t, 1, mask, f, geom_for_axis(1, sx2, sy2, 2 * c), border, border, dc, s, /*pdl=*/true);
      if (r) return r;
      // cells 2l and 2l + 1 along the last axis: one doubled slice (3-D) or row (2-D) apart
      const int64_t step = ndim == 3 ? 4 * sx * sy : 2 * sx;
      for (int h = 0; h < 2; ++h) {
        voxel_graph_gather_kernel<<<blocks(c * plane), threads, 0, s>>>(f + h * step, slots.plane(slot, cells + h), sx,
                                                                          cy, cz, 2, 4 * sx, 8 * sx * sy, 0);
        CUDA_TRY(cudaGetLastError());
      }
      return 0;
    };
    steps.download = [&](int k, int slot, cudaStream_t s) {
      const int r = download_box(two.slab(out, k, sizeof(float)), slots.plane(slot, cells), device, s);
      return r ? r : download_box(two.slab(odd_cells.get(), k, sizeof(float)), slots.plane(slot, cells + 1), device, s);
    };
  });
  if (rc) return rc;
  return run_phase(dc, device, two.p2, label_bytes + 1, planes2, [&](const ChunkSlots& slots, PipelineSteps& steps) {
    steps.item = "phase-2 chunk";
    steps.upload_writes_results = true;            // cell 2l goes up into the volume the result comes down from
    steps.upload = [&](int k, int slot, cudaStream_t s) {
      int r = upload_box(slots.labels[slot], two.lines(labels, k, label_bytes), device, s);
      if (!r) r = upload_box(static_cast<char*>(slots.labels[slot]) + slots.vox * label_bytes, two.lines(graph, k, 1),
                             device, s);
      if (!r) r = upload_box(slots.plane(slot, 2), two.lines(out, k, sizeof(float)), device, s);
      return r ? r : upload_box(slots.plane(slot, 3), two.lines(odd_cells.get(), k, sizeof(float)), device, s);
    };
    steps.passes = [&](int k, int slot, cudaStream_t s) {
      const int64_t c = two.p2.size(k), bp = two.unit * c;  // bp: the box's voxels per index of the last axis
      const uint8_t* gr = reinterpret_cast<const uint8_t*>(slots.labels[slot]) + slots.vox * label_bytes;
      float* f = slots.plane(slot, 0);
      uint8_t* mask = slots.plane<uint8_t>(slot, 4);
      int r = with_label_width(label_bytes, [&](auto b) {
        voxel_graph_lines_kernel<b><<<blocks(bp * n_last), threads, 0, s>>>(
            slots.labels[slot], gr, slots.plane(slot, 2), slots.plane(slot, 3), bp, n_last, ndim == 3 ? 0x10 : 0x04,
            border, as_float, f, mask);
        CUDA_TRY(cudaGetLastError());
        return 0;
      });
      const LineGeom g = ndim == 3 ? geom_for_axis(2, sx, c, sz2) : geom_for_axis(1, c, sy2, 1);
      if (!r) r = later_pass(t, last, mask, f, g, border, border, dc, s, /*pdl=*/false);
      if (r) return r;
      voxel_graph_gather_kernel<<<blocks(bp * n_last), threads, 0, s>>>(f, slots.plane(slot, 2), bp, n_last, 1, 1,
                                                                         2 * bp, 0, (flags & EDTB200_SQRT) ? 1 : 0);
      CUDA_TRY(cudaGetLastError());
      return 0;
    };
    steps.download = [&](int k, int slot, cudaStream_t s) {
      return download_box(two.lines(out, k, sizeof(float)), slots.plane(slot, 2), device, s);
    };
  });
}

int edtb200_pass_first(const void* labels_dev, int label_bytes, int64_t sx, int64_t sy, int64_t sz,
                       float wx, int black_border, int flags, float* f_dev, int device, void* stream) {
  int rc = check_dims(label_bytes, 3, sx, sy, sz);
  if (rc) return rc;
  if (sx * sy * sz == 0) return 0;
  if (!labels_dev || !f_dev) return fail(EDTB200_EINVAL, "null pointer");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  // EDTB200_SIGNED only makes the background an ordinary label here: no sign is applied
  const int kflags = kernel_flags(flags, /*first=*/true, /*last=*/true) & ~edtb200::kNegate;
  return dispatch_first(label_bytes, labels_dev, f_dev, sy * sz, sx, wx, black_border != 0, kflags, *dc,
                        static_cast<cudaStream_t>(stream));
}

// The arithmetic of a later pass with weight w along lines of n rows over `count` samples the caller
// gave (edtb200_pass_later, edtb200_pass_window): one reduction over them on s, and a wait for it,
// tells whether the candidate sums are exact in double, and whether the integer hull tests apply.
int caller_samples_arith(const float* f_dev, int64_t count, float w, int64_t n, DeviceCache& dc, cudaStream_t s,
                         PassArith* arith) {
  const int init[2] = {0, 1024};
  int range[2] = {0, 1024};
  {
    Scratch range_dev;                                           // freed before the wait below
    CUDA_TRY(range_dev.alloc(dc, 2 * sizeof(int), s));
    CUDA_TRY(cudaMemcpyAsync(range_dev.get(), init, sizeof(init), cudaMemcpyHostToDevice, s));
    int64_t blocks = (count + 255) / 256;
    if (blocks > (int64_t)dc.sm_count * 8) blocks = (int64_t)dc.sm_count * 8;
    sample_range_kernel<<<(unsigned)blocks, 256, 0, s>>>(f_dev, count, range_dev.get<int>());
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(range, range_dev.get(), sizeof(range), cudaMemcpyDeviceToHost, s));
  }
  CUDA_TRY(cudaStreamSynchronize(s));
  float fmax;
  memcpy(&fmax, &range[0], sizeof(float));
  *arith = sampled_arith(fmax, range[1], w, n);
  return 0;
}

int edtb200_pass_later(const void* labels_dev, int label_bytes, int axis, int64_t sx, int64_t sy, int64_t sz,
                       float w, int border_lo, int border_hi, int flags, float* f_dev, int device,
                       void* stream) {
  int rc = check_dims(label_bytes, 3, sx, sy, sz);
  if (rc) return rc;
  if (axis != 1 && axis != 2) return fail(EDTB200_EINVAL, "axis must be 1 (Y) or 2 (Z)");
  if (sx * sy * sz == 0) return 0;
  if (!labels_dev || !f_dev) return fail(EDTB200_EINVAL, "null pointer");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const edtb200::LineGeom g = geom_for_axis(axis, sx, sy, sz);
  PassArith arith;
  rc = caller_samples_arith(f_dev, sx * sy * sz, w, g.n, *dc, s, &arith);
  if (rc) return rc;
  return dispatch_later(label_bytes, labels_dev, f_dev, g, w, border_lo != 0, border_hi != 0,
                        kernel_flags(flags, /*first=*/false, /*last=*/true), arith, *dc, s, /*pdl=*/false);
}

int edtb200_pass_window(const void* labels_dev, int label_bytes, int axis, int64_t sx, int64_t sy, int64_t sz,
                        float w, int border_lo, int border_hi, int flags, double max_distance, const float* fin_dev,
                        float* fout_dev, int* codes_dev, int device, void* stream) {
  int rc = check_dims(label_bytes, 3, sx, sy, sz);
  if (rc) return rc;
  if (axis != 1 && axis != 2) return fail(EDTB200_EINVAL, "axis must be 1 (Y) or 2 (Z)");
  if ((rc = check_weights(1, &w))) return rc;
  if (!(max_distance >= 0.0)) return fail(EDTB200_EINVAL, "max_distance must be zero or more (got %g)", max_distance);
  const BoundedPlan bp = window_pass_plan(w, max_distance);
  if (bp.radius[0] > kWindowRadiusLimit)
    return fail(EDTB200_EINVAL, "window radius %lld out of range", (long long)bp.radius[0]);
  const int64_t count = sx * sy * sz;
  if (count == 0) return 0;
  if (!labels_dev || !fin_dev || !fout_dev) return fail(EDTB200_EINVAL, "null pointer");
  const size_t bytes = sizeof(float) * (size_t)count;
  if (overlaps(fin_dev, bytes, fout_dev, bytes) || (codes_dev && (overlaps(codes_dev, bytes, fin_dev, bytes) ||
                                                                  overlaps(codes_dev, bytes, fout_dev, bytes))))
    return fail(EDTB200_EINVAL, "fin, fout and codes must not overlap");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const edtb200::LineGeom g = geom_for_axis(axis, sx, sy, sz);
  PassArith arith;
  rc = caller_samples_arith(fin_dev, count, w, g.n, *dc, s, &arith);
  if (rc) return rc;
  return with_label_width(label_bytes, [&](auto b) {
    return launch_later_window<b>(labels_dev, fin_dev, fout_dev, codes_dev, g, w, (int)bp.radius[0], border_lo != 0,
                                  border_hi != 0, kernel_flags(flags, /*first=*/false, /*last=*/true), arith,
                                  bp.bound, *dc, s);
  });
}

int edtb200_noise_planes(const void* labels_dev, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                         int64_t count, float wx, float wy, float wz, int black_border, int flags, int passes,
                         int nchunks, int ctas, float* f_dev, uint32_t* planes_dev, int* info, int device,
                         void* stream) {
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (label_bytes < 4) return fail(EDTB200_EINVAL, "the run-start planes need labels of 4 or 8 bytes (got %d)", label_bytes);
  if (ndim < 2) return fail(EDTB200_EINVAL, "the run-start planes need 2-D or 3-D volumes (got ndim %d)", ndim);
  if (count < 1) return fail(EDTB200_EINVAL, "count must be 1 or more (got %lld)", (long long)count);
  if ((rc = check_stack(sx * sy * sz, count, 1))) return rc;
  const float w[3] = {wx, wy, wz};
  if ((rc = check_weights(ndim, w))) return rc;
  if (flags & EDTB200_SIGNED) return fail(EDTB200_EINVAL, "a signed transform (EDTB200_SIGNED) takes no run-start planes");
  if (flags & ~EDTB200_SQRT) return fail(EDTB200_EINVAL, "flags may only hold EDTB200_SQRT (got %d)", flags);
  if (passes != 1 && passes != 2) return fail(EDTB200_EINVAL, "passes must be 1 or 2 (got %d)", passes);
  if (sx > 512 || sx % 4 != 0)
    return fail(EDTB200_EINVAL, "the run-start planes need rows of at most 512 voxels, a multiple of 4 (got %lld)",
                (long long)sx);
  if (sz * count > 0x7fffffffLL || sy > 0x3fffffffLL)
    return fail(EDTB200_EINVAL, "more slices or rows than the plane-writing X pass counts in 32 bits");
  if (nchunks < 0 || nchunks > sy)
    return fail(EDTB200_EINVAL, "nchunks must be 0 or 1..sy = %lld (got %d)", (long long)sy, nchunks);
  if (ctas < 0 || (ctas > 0 && nchunks == 0))
    return fail(EDTB200_EINVAL, "ctas must be 0, or 1..items with nchunks given (got %d)", ctas);
  if (ctas > 0) {
    using edtb200::kPlaneWarps;
    const int64_t items = ndim == 3 ? edtb200::march_items<kPlaneWarps, 2>(sz * count, nchunks)
                                    : edtb200::march_items<kPlaneWarps, 1>(count, nchunks);
    if (ctas > items) return fail(EDTB200_EINVAL, "ctas must be 0 or 1..items = %lld (got %d)", (long long)items, ctas);
  }
  if (sx * sy * sz == 0) return 0;
  if (!labels_dev || !f_dev || !planes_dev || !info) return fail(EDTB200_EINVAL, "null pointer");
  if (!first_is_vec(labels_dev, label_bytes, f_dev, sx) || reinterpret_cast<uintptr_t>(planes_dev) % 4 != 0)
    return fail(EDTB200_EINVAL, "labels, distances and planes must be aligned for vector access");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const Transform t{label_bytes, ndim, flags, black_border != 0, {wx, wy, wz}, {sx, sy, sz}};
  // the plan of the second call on label noise; the X pass writes the planes whatever the later passes take
  NoisePlan np = noise_plan(t, count, labels_dev, f_dev, *dc, /*noise=*/1);
  if (passes == 2 && !np.planes)
    return fail(EDTB200_EINVAL, "the transform takes no run-start planes for these extents and weights");
  np.planes = ndim - 1;
  RunPlanes rp;
  arm_run_planes(rp, np, t, planes_dev, sy, sz, count);
  PlanesMarch march;
  march.want_chunks = nchunks;
  march.want_ctas = ctas;
  rc = x_pass(t, labels_dev, f_dev, sy * sz * count, *dc, s, &rp, &march);
  if (!rc && passes == 2)
    rc = later_pass(t, 1, labels_dev, f_dev, geom_for_axis(1, sx, sy, sz, count), t.border, t.border, *dc, s,
                    /*pdl=*/true, &rp);
  if (rc) return rc;
  const int v[10] = {label_bytes, march.k, march.plain, march.planes, (int)march.nchunks, (int)march.items,
                     (int)march.grid, passes == 2 && np.reads[1], passes == 2 && np.later[1].settled,
                     passes == 2 && np.refresh};
  memcpy(info, v, sizeof(v));
  return 0;
}

int edtb200_last_later_launch(int* info) {
  if (!info) return fail(EDTB200_EINVAL, "null pointer");
  const LaterLaunch& l = g_last_later;
  if (l.kernel < 0) return fail(EDTB200_EINVAL, "no later-axis pass has been launched on this thread");
  const int v[9] = {l.kernel, l.tx, l.tma, l.wide, l.ctas, l.int_hull, l.epilogue, l.all_double, l.settled};
  memcpy(info, v, sizeof(v));
  return 0;
}

int edtb200_slab_face_runs(const void* labels_dev, int label_bytes, int64_t sx, int64_t sy, int64_t sz,
                           int high_face, int halo, int flags, unsigned char* m_dev, int* overflow_dev,
                           int device, void* stream_v) {
  int rc = check_dims(label_bytes, 3, sx, sy, sz);
  if (rc) return rc;
  if (halo < 1 || halo > 254) return fail(EDTB200_EINVAL, "halo must be in 1..254");
  if (sx * sy * sz == 0) return 0;
  if (!labels_dev || !m_dev || !overflow_dev) return fail(EDTB200_EINVAL, "null pointer");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int64_t plane = sx * sy;
  const unsigned blocks = (unsigned)((plane + 255) / 256);
  const int zl = (flags & EDTB200_SIGNED) ? 1 : 0;
  using namespace edtb200;
  return with_label_width(label_bytes, [&](auto b) {
    using LT = typename LabelOf<b>::type;
    face_runs_kernel<b><<<blocks, 256, 0, stream>>>(static_cast<const LT*>(labels_dev), plane, (int)sz, high_face,
                                                    halo, zl, m_dev, overflow_dev);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

int edtb200_slab_pack(const void* src_dev, void* dst_dev, int64_t zc, int64_t sy, int64_t row_bytes, int parts,
                      const int64_t* y_start, int unpack, int device, void* stream_v) {
  if (zc < 0 || sy < 0 || row_bytes < 0) return fail(EDTB200_EINVAL, "negative extent");
  if (parts < 1 || parts > 64) return fail(EDTB200_EINVAL, "parts must be in 1..64");
  if (!y_start) return fail(EDTB200_EINVAL, "null pointer");
  edtb200::SlabParts sp;
  sp.n = parts;
  for (int i = 0; i <= parts; ++i) {
    sp.start[i] = y_start[i];
    if ((i == 0 && y_start[i] != 0) || (i > 0 && y_start[i] < y_start[i - 1]))
      return fail(EDTB200_EINVAL, "y_start must rise from 0 to sy");
  }
  if (y_start[parts] != sy) return fail(EDTB200_EINVAL, "y_start must rise from 0 to sy");
  if (zc * sy * row_bytes == 0) return 0;
  if (!src_dev || !dst_dev) return fail(EDTB200_EINVAL, "null pointer");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  int rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int vec16 = (row_bytes % 16 == 0 && reinterpret_cast<uintptr_t>(src_dev) % 16 == 0 &&
                     reinterpret_cast<uintptr_t>(dst_dev) % 16 == 0) ? 1 : 0;
  const int64_t rows = zc * sy;
  const unsigned blocks = (unsigned)std::min<int64_t>(rows, (int64_t)dc->sm_count * 32);
  const unsigned char* a = static_cast<const unsigned char*>(src_dev);
  unsigned char* b = static_cast<unsigned char*>(dst_dev);
  if (unpack) edtb200::slab_pack_kernel<true><<<blocks, 256, 0, stream>>>(a, b, zc, sy, row_bytes, vec16, sp);
  else edtb200::slab_pack_kernel<false><<<blocks, 256, 0, stream>>>(a, b, zc, sy, row_bytes, vec16, sp);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int edtb200_slab_face_fixup(const void* labels_dev, int label_bytes, int64_t sx, int64_t sy, int64_t sz,
                            int high_face, int halo, float wz, int flags, const void* nb_label_dev,
                            const unsigned char* nb_m_dev, const float* nb_f_dev, float* f_dev, int* inexact_dev,
                            int device, void* stream_v) {
  int rc = check_dims(label_bytes, 3, sx, sy, sz);
  if (rc) return rc;
  if (halo < 1 || halo > 254) return fail(EDTB200_EINVAL, "halo must be in 1..254");
  if (sx * sy * sz == 0) return 0;
  if (!labels_dev || !nb_label_dev || !nb_m_dev || !nb_f_dev || !f_dev) return fail(EDTB200_EINVAL, "null pointer");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int64_t plane = sx * sy;
  const unsigned blocks = (unsigned)((plane + 255) / 256);
  using namespace edtb200;
  // the last pass's store, on a transform whose first pass may have treated background as a label
  const int kflags = kernel_flags(flags, /*first=*/true, /*last=*/true);
  const float w2 = wz * wz;
  return with_label_width(label_bytes, [&](auto b) {
    using LT = typename LabelOf<b>::type;
    face_fixup_kernel<b><<<blocks, 256, 0, stream>>>(static_cast<const LT*>(labels_dev), f_dev, plane, (int)sz,
                                                     high_face, halo, w2, static_cast<const LT*>(nb_label_dev),
                                                     nb_m_dev, nb_f_dev, kflags, inexact_dev);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

// ---- one host volume on several GPUs of this process ---------------------------------------
// Z slabs for the X and Y passes, Y slabs (whole z lines) for the Z pass: between the two the
// distances and labels are re-partitioned by peer-to-peer 3-D copies over NVLink, so the result is
// exact for any input with no halo and no verdict -- for a HOST volume the PCIe copies dominate
// anyway and every GPU brings its own link.  One host thread per device; the threads meet at two
// barriers (after the Y passes, after the Z passes), the devices through events.
namespace {

struct MultiBarrier {
  std::mutex m;
  std::condition_variable cv;
  int waiting = 0, generation = 0, parties = 0, failed = 0;
  // returns the failure code agreed by all parties (0 = go on)
  int arrive(int my_rc) {
    std::unique_lock<std::mutex> l(m);
    if (my_rc && !failed) failed = my_rc;
    const int gen = generation;
    if (++waiting == parties) { waiting = 0; ++generation; cv.notify_all(); }
    else cv.wait(l, [&] { return generation != gen; });
    return failed;
  }
};

struct MultiPart {
  int device = 0;
  int64_t z0 = 0, zc = 0, y0 = 0, yc = 0;
  void* lz = nullptr; float* fz = nullptr; void* ly = nullptr; float* fy = nullptr;
  cudaStream_t stream = nullptr;
  cudaEvent_t after_y = nullptr, after_z = nullptr;
  char error[256] = "";
};

cudaError_t copy_box(void* dst, size_t dst_row_bytes, int64_t dst_rows_per_slice, int dst_dev, int64_t dx_bytes,
                     int64_t dy, int64_t dz, const void* src, size_t src_row_bytes, int64_t src_rows_per_slice,
                     int src_dev, int64_t sx_bytes, int64_t sy0, int64_t sz0, size_t width_bytes, int64_t height,
                     int64_t depth, cudaStream_t stream) {
  cudaMemcpy3DPeerParms p;
  memset(&p, 0, sizeof(p));
  p.srcDevice = src_dev;
  p.dstDevice = dst_dev;
  p.srcPtr = make_cudaPitchedPtr(const_cast<void*>(src), src_row_bytes, src_row_bytes, (size_t)src_rows_per_slice);
  p.dstPtr = make_cudaPitchedPtr(dst, dst_row_bytes, dst_row_bytes, (size_t)dst_rows_per_slice);
  p.srcPos = make_cudaPos((size_t)sx_bytes, (size_t)sy0, (size_t)sz0);
  p.dstPos = make_cudaPos((size_t)dx_bytes, (size_t)dy, (size_t)dz);
  p.extent = make_cudaExtent(width_bytes, (size_t)height, (size_t)depth);
  return cudaMemcpy3DPeerAsync(&p, stream);
}

}  // namespace

int edtb200_transform_multi(const void* labels, int label_bytes, int ndim, int64_t sx, int64_t sy, int64_t sz,
                            float wx, float wy, float wz, int black_border, int flags, float* out,
                            const int* devices, int ndevices) {
  if (!devices || ndevices < 1) return fail(EDTB200_EINVAL, "no devices given");
  if (flags & (EDTB200_LABELS_ON_DEVICE | EDTB200_OUT_ON_DEVICE))
    return fail(EDTB200_EINVAL, "edtb200_transform_multi splits a HOST volume over the devices");
  int rc = check_dims(label_bytes, ndim, sx, sy, sz);
  if (rc) return rc;
  if (sx * sy * sz == 0) return 0;
  if (!labels || !out) return fail(EDTB200_EINVAL, "null pointer");
  for (int i = 0; i < ndevices; ++i)
    for (int j = 0; j < i; ++j)
      if (devices[i] == devices[j]) return fail(EDTB200_EINVAL, "device %d listed twice", devices[i]);
  int G = ndevices;
  if (ndim < 3) G = 1;
  if (G > sz) G = (int)sz;
  if (G > sy) G = (int)sy;
  if (G <= 1)
    return edtb200_transform(labels, label_bytes, ndim, sx, sy, sz, wx, wy, wz, black_border, flags, out, devices[0],
                             nullptr);

  const int border = black_border != 0;
  const Transform t{label_bytes, ndim, flags, border, {wx, wy, wz}, {sx, sy, sz}};
  std::vector<MultiPart> parts(G);
  for (int d = 0; d < G; ++d) {
    MultiPart& p = parts[d];
    p.device = devices[d];
    p.z0 = sz * d / G; p.zc = sz * (d + 1) / G - p.z0;
    p.y0 = sy * d / G; p.yc = sy * (d + 1) / G - p.y0;
  }
  MultiBarrier barrier;
  barrier.parties = G;
  const size_t row_l = (size_t)sx * label_bytes, row_f = (size_t)sx * sizeof(float);

  auto worker = [&](int d) -> int {
    MultiPart& me = parts[d];
    DeviceGuard restore_device;
    DeviceCache* dc = nullptr;
    int wrc = probe(me.device, &dc);
    std::unique_lock<std::mutex> host_call;
    auto note = [&](int code) { snprintf(me.error, sizeof(me.error), "device %d: %.200s", me.device, g_error); return code; };
    #define MULTI_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess && !wrc) { \
        wrc = fail(e_ == cudaErrorMemoryAllocation ? EDTB200_ENOMEM : EDTB200_ECUDA, "%s: %s", #expr, \
                   cudaGetErrorString(e_)); note(wrc); } } while (0)
    if (!wrc) {
      host_call = std::unique_lock<std::mutex>(dc->host_call);
      for (int o = 0; o < G; ++o)                                 // direct NVLink copies where possible
        if (o != d) { cudaDeviceEnablePeerAccess(parts[o].device, 0); cudaGetLastError(); }
      MULTI_TRY(private_stream(*dc));
      me.stream = dc->stream;
      MULTI_TRY(cudaEventCreateWithFlags(&me.after_y, cudaEventDisableTiming));
      MULTI_TRY(cudaEventCreateWithFlags(&me.after_z, cudaEventDisableTiming));
      const size_t nz_vox = (size_t)sx * sy * me.zc, ny_vox = (size_t)sx * me.yc * sz;
      MULTI_TRY(scratch_alloc(*dc, &me.lz, nz_vox * label_bytes, me.stream));
      MULTI_TRY(scratch_alloc(*dc, reinterpret_cast<void**>(&me.fz), nz_vox * sizeof(float), me.stream));
      MULTI_TRY(scratch_alloc(*dc, &me.ly, ny_vox * label_bytes, me.stream));
      MULTI_TRY(scratch_alloc(*dc, reinterpret_cast<void**>(&me.fy), ny_vox * sizeof(float), me.stream));
    } else {
      note(wrc);
    }
    // ---- phase A: my Z slab up, X and Y passes ----
    if (!wrc) {
      const char* src = static_cast<const char*>(labels) + (size_t)me.z0 * sy * row_l;
      wrc = upload(me.lz, src, (size_t)sx * sy * me.zc * label_bytes, me.device, me.stream);
      if (!wrc) wrc = x_pass(t, me.lz, me.fz, sy * me.zc, *dc, me.stream);
      if (!wrc) wrc = later_pass(t, 1, me.lz, me.fz, geom_for_axis(1, sx, sy, me.zc), border, border, *dc, me.stream,
                                 /*pdl=*/true);
      if (wrc) note(wrc);
      MULTI_TRY(cudaEventRecord(me.after_y, me.stream));
    }
    int agreed = barrier.arrive(wrc);
    // ---- phase B: gather my Y slab (whole z lines) from every Z slab, Z pass ----
    if (!agreed) {
      for (int o = 0; o < G && !wrc; ++o) {
        const MultiPart& src = parts[o];
        MULTI_TRY(cudaStreamWaitEvent(me.stream, src.after_y, 0));
        MULTI_TRY(copy_box(me.fy, row_f, me.yc, me.device, 0, 0, src.z0, src.fz, row_f, sy, src.device, 0, me.y0, 0,
                           row_f, me.yc, src.zc, me.stream));
        MULTI_TRY(copy_box(me.ly, row_l, me.yc, me.device, 0, 0, src.z0, src.lz, row_l, sy, src.device, 0, me.y0, 0,
                           row_l, me.yc, src.zc, me.stream));
      }
      if (!wrc) {
        wrc = later_pass(t, 2, me.ly, me.fy, geom_for_axis(2, sx, me.yc, sz), border, border, *dc, me.stream,
                         /*pdl=*/false);
        if (wrc) note(wrc);
      }
      MULTI_TRY(cudaEventRecord(me.after_z, me.stream));
    }
    agreed = barrier.arrive(wrc);
    // ---- phase C: my Z slab of the result back from every Y slab, then down to the host ----
    if (!agreed) {
      for (int o = 0; o < G && !wrc; ++o) {
        const MultiPart& src = parts[o];
        MULTI_TRY(cudaStreamWaitEvent(me.stream, src.after_z, 0));
        MULTI_TRY(copy_box(me.fz, row_f, sy, me.device, 0, src.y0, 0, src.fy, row_f, src.yc, src.device, 0, 0, me.z0,
                           row_f, src.yc, me.zc, me.stream));
      }
      if (!wrc) {
        char* dst = reinterpret_cast<char*>(out) + (size_t)me.z0 * sy * row_f;
        wrc = download(dst, me.fz, (size_t)sx * sy * me.zc * sizeof(float), me.device, me.stream);
        if (wrc) note(wrc);
      }
    }
    if (me.stream) cudaStreamSynchronize(me.stream);
    agreed = barrier.arrive(wrc);                                 // nobody frees what a peer may still read
    void* all[] = {me.lz, me.fz, me.ly, me.fy};
    for (void* q : all) if (q) cudaFreeAsync(q, me.stream);
    if (me.after_y) cudaEventDestroy(me.after_y);
    if (me.after_z) cudaEventDestroy(me.after_z);
    cudaGetLastError();
    #undef MULTI_TRY
    return wrc ? wrc : agreed;
  };

  std::vector<int> rcs(G, 0);
  std::vector<std::thread> threads;
  for (int d = 1; d < G; ++d) threads.emplace_back([&, d] { rcs[d] = worker(d); });
  rcs[0] = worker(0);
  for (auto& t : threads) t.join();
  for (int d = 0; d < G; ++d)
    if (rcs[d] && parts[d].error[0]) return fail(rcs[d], "%s", parts[d].error);
  for (int d = 0; d < G; ++d)
    if (rcs[d]) return fail(rcs[d], "multi-device transform failed on device %d", parts[d].device);
  return 0;
}

int64_t edtb200_slab_stage_bytes(int64_t sx, int64_t sy, int label_bytes, int halo) {
  if (sx <= 0 || sy <= 0 || halo < 1 || halo > 254 ||
      !(label_bytes == 1 || label_bytes == 2 || label_bytes == 4 || label_bytes == 8))
    return -1;
  return (int64_t)edtb200::slab_stage_layout(sx * sy, label_bytes, halo).total_bytes;
}

int edtb200_slab_step(const void* labels_dev, int label_bytes, int64_t sx, int64_t sy, int64_t sz,
                      float wx, float wy, float wz, int black_border, int has_lo, int has_hi, int flags,
                      float* f_dev, int halo, void* sym_self, void* sym_lo, void* sym_hi,
                      unsigned long long step, int* status_dev, int device, void* stream_v) {
  using namespace edtb200;
  int rc = check_dims(label_bytes, 3, sx, sy, sz);
  if (rc) return rc;
  if (halo < 1 || halo > 254) return fail(EDTB200_EINVAL, "halo must be in 1..254");
  if (sz <= halo && (has_lo || has_hi)) return fail(EDTB200_EINVAL, "the slab must be deeper than the halo");
  if (!labels_dev || !f_dev || !sym_self || !status_dev) return fail(EDTB200_EINVAL, "null pointer");
  if ((has_lo && !sym_lo) || (has_hi && !sym_hi)) return fail(EDTB200_EINVAL, "missing neighbour buffer");
  if (step == 0) return fail(EDTB200_EINVAL, "steps are counted from 1");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int border = black_border != 0;
  const Transform t{label_bytes, 3, flags, border, {wx, wy, wz}, {sx, sy, sz}};

  // verbose: the device time of every phase of the step, with the launches serialised
  StepTimer timer(stream);
  const bool verbose = timer.on();
  timer.stamp();
  mark_pass(0, stream);              // per-pass events for bench.py (edtb200_profile_passes), as in run_passes
  // X and Y passes: slab-local
  nvtx_push("edt.x");
  rc = x_pass(t, labels_dev, f_dev, sy * sz, *dc, stream);
  nvtx_pop();
  if (rc) return rc;
  timer.stamp();
  mark_pass(1, stream);
  nvtx_push("edt.y");
  rc = later_pass(t, 1, labels_dev, f_dev, geom_for_axis(1, sx, sy, sz), border, border, *dc, stream,
                  /*pdl=*/!verbose);
  nvtx_pop();
  if (rc) return rc;
  timer.stamp();

  const int64_t plane = sx * sy;
  const SlabStageLayout L = slab_stage_layout(plane, label_bytes, halo);
  unsigned char* self = static_cast<unsigned char*>(sym_self);
  unsigned char* lo = static_cast<unsigned char*>(sym_lo);
  unsigned char* hi = static_cast<unsigned char*>(sym_hi);
  const int parity = (int)(step & 1ull);
  const dim3 grid((unsigned)((plane + 255) / 256), 2);
  if (has_lo || has_hi) {
    nvtx_push("edt.halo.stage");
    unsigned char* set = self + (size_t)parity * L.set_bytes;
    // I am the HIGH neighbour of the rank below me and the LOW neighbour of the rank above me
    unsigned long long* flag_in_lo_peer = has_lo ? reinterpret_cast<unsigned long long*>(lo + L.flag_from_hi) : nullptr;
    unsigned long long* flag_in_hi_peer = has_hi ? reinterpret_cast<unsigned long long*>(hi + L.flag_from_lo) : nullptr;
    unsigned int* counter = reinterpret_cast<unsigned int*>(self + L.counter);
    rc = with_label_width(label_bytes, [&](auto b) {
      using LT = typename LabelOf<b>::type;
      slab_stage_kernel<b><<<grid, 256, 0, stream>>>(static_cast<const LT*>(labels_dev), f_dev, plane, (int)sz, halo,
                                                     has_lo, has_hi, set, L, step, flag_in_lo_peer, flag_in_hi_peer,
                                                     counter);
      CUDA_TRY(cudaGetLastError());
      return 0;
    });
    if (rc) return rc;
    nvtx_pop();
  }

  timer.stamp();
  mark_pass(2, stream);              // "second pass" = Y plus the face staging kernel
  // Z pass on the slab, interior faces open
  nvtx_push("edt.z");
  rc = later_pass(t, 2, labels_dev, f_dev, geom_for_axis(2, sx, sy, sz), border && !has_lo, border && !has_hi, *dc,
                  stream, /*pdl=*/!verbose && (has_lo || has_hi));
  nvtx_pop();
  if (rc) return rc;

  timer.stamp();
  mark_pass(3, stream);
  if (has_lo || has_hi) {
    nvtx_push("edt.halo.fixup");
    const int kflags = kernel_flags(flags, /*first=*/true, /*last=*/true);
    const float w2 = wz * wz;
    const unsigned char* set_lo = has_lo ? lo + (size_t)parity * L.set_bytes : nullptr;
    const unsigned char* set_hi = has_hi ? hi + (size_t)parity * L.set_bytes : nullptr;
    const unsigned long long* flag_from_lo = reinterpret_cast<const unsigned long long*>(self + L.flag_from_lo);
    const unsigned long long* flag_from_hi = reinterpret_cast<const unsigned long long*>(self + L.flag_from_hi);
    cudaLaunchConfig_t fcfg = {};
    fcfg.gridDim = dim3(grid.x);             // both faces of a line in one thread, low face first
    fcfg.blockDim = dim3(256); fcfg.dynamicSmemBytes = 0; fcfg.stream = stream;
    cudaLaunchAttribute fattr[1];
    fattr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    fattr[0].val.programmaticStreamSerializationAllowed = 1;
    fcfg.attrs = fattr;
    fcfg.numAttrs = verbose ? 0 : 1;         // behind our own Z pass, which triggers its dependents early
    rc = with_label_width(label_bytes, [&](auto b) {
      using LT = typename LabelOf<b>::type;
      CUDA_TRY(cudaLaunchKernelEx(&fcfg, slab_fixup_kernel<b>, static_cast<const LT*>(labels_dev), f_dev, plane,
                                  (int)sz, halo, w2, has_lo, has_hi, set_lo, set_hi, L, step, flag_from_lo,
                                  flag_from_hi, kflags, status_dev));
      CUDA_TRY(cudaGetLastError());
      return 0;
    });
    if (rc) return rc;
    nvtx_pop();
  }
  timer.stamp();
  if (verbose) {
    float ms[5] = {0, 0, 0, 0, 0};
    if (timer.synchronize())
      for (int i = 0; i < 5; ++i) ms[i] = timer.ms(i, i + 1);
    fprintf(stderr, "[edt_b200] slab step %llu dev %d: x %.3f  y %.3f  stage %.3f  z %.3f  fixup %.3f ms\n", step, device,
            ms[0], ms[1], ms[2], ms[3], ms[4]);
  }
  return 0;
}

int edtb200_label_stats(const void* labels_dev, int label_bytes, const float* dt_dev, int64_t sx, int64_t sy,
                        int64_t sz, int capacity, unsigned long long* keys_dev, unsigned long long* count_dev,
                        float* max_dev, long long* argmax_dev, int* box_dev, int* overflow_dev, int device,
                        void* stream_v) {
  using namespace edtb200;
  int rc = check_dims(label_bytes, 3, sx, sy, sz);
  if (rc) return rc;
  if (capacity < 2 || (capacity & (capacity - 1))) return fail(EDTB200_EINVAL, "capacity must be a power of two");
  if (!labels_dev || !dt_dev || !keys_dev || !count_dev || !max_dev || !argmax_dev || !box_dev || !overflow_dev)
    return fail(EDTB200_EINVAL, "null pointer");
  if (sx > 0x7fffffff || sy > 0x7fffffff || sz > 0x7fffffff) return fail(EDTB200_ELIMIT, "axis too long");
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  LabelTable t;
  t.keys = keys_dev; t.count = count_dev; t.maxbits = reinterpret_cast<unsigned int*>(max_dev);
  t.argmax = argmax_dev; t.box = box_dev; t.capacity = capacity; t.overflow = overflow_dev;
  label_table_init_kernel<<<(capacity + 255) / 256, 256, 0, stream>>>(t);
  CUDA_TRY(cudaMemsetAsync(overflow_dev, 0, sizeof(int), stream));
  const int64_t total = sx * sy * sz;
  if (total > 0) {
    const unsigned blocks = (unsigned)std::min<int64_t>((total + 255) / 256, (int64_t)dc->sm_count * 16);
    rc = with_label_width(label_bytes, [&](auto b) {
      using LT = typename LabelOf<b>::type;
      label_stats_kernel<b><<<blocks, 256, 0, stream>>>(static_cast<const LT*>(labels_dev), dt_dev, total, (int)sx,
                                                        (int)sy, t);
      label_argmax_kernel<b><<<blocks, 256, 0, stream>>>(static_cast<const LT*>(labels_dev), dt_dev, total, t);
      return 0;
    });
    if (rc) return rc;
  }
  label_table_finish_kernel<<<(capacity + 255) / 256, 256, 0, stream>>>(t);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

int edtb200_label_extract(const void* labels_dev, int label_bytes, const float* dt_dev, int64_t sx, int64_t sy,
                          int64_t sz, unsigned long long key, const int* box, int erase, float* out_dev,
                          int device, void* stream_v) {
  using namespace edtb200;
  int rc = check_dims(label_bytes, 3, sx, sy, sz);
  if (rc) return rc;
  if (!labels_dev || !dt_dev || !out_dev) return fail(EDTB200_EINVAL, "null pointer");
  if (sx > 0x7fffffff || sy > 0x7fffffff || sz > 0x7fffffff) return fail(EDTB200_ELIMIT, "axis too long");
  int b[6] = {0, 0, 0, (int)sx - 1, (int)sy - 1, (int)sz - 1};
  if (box) for (int i = 0; i < 6; ++i) b[i] = box[i];
  if (b[0] < 0 || b[1] < 0 || b[2] < 0 || b[3] >= sx || b[4] >= sy || b[5] >= sz)
    return fail(EDTB200_EINVAL, "box outside the volume");
  if (b[3] < b[0] || b[4] < b[1] || b[5] < b[2]) return 0;             // empty box
  DeviceGuard restore_device;
  DeviceCache* dc = nullptr;
  rc = probe(device, &dc);
  if (rc) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int bx = b[3] - b[0] + 1, by = b[4] - b[1] + 1, bz = b[5] - b[2] + 1;
  const int64_t rows = (int64_t)by * bz;
  const unsigned blocks = (unsigned)std::min<int64_t>((rows + 7) / 8, (int64_t)dc->sm_count * 16);
  return with_label_width(label_bytes, [&](auto w) {
    using LT = typename LabelOf<w>::type;
    label_extract_kernel<w><<<blocks, 256, 0, stream>>>(static_cast<const LT*>(labels_dev), dt_dev, out_dev, (int)sx,
                                                        (int)sy, b[0], b[1], b[2], bx, by, bz, key, erase);
    CUDA_TRY(cudaGetLastError());
    return 0;
  });
}

void* edtb200_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (bytes == 0 || cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}

void edtb200_host_free(void* p) {
  if (p) { cudaFreeHost(p); cudaGetLastError(); }
}

int edtb200_profile_passes(int enable) {
  g_profile = enable != 0;
  if (enable) g_pass_seq = 0;
  return 0;
}

int edtb200_pass_ms(int steps_back, float* ms3) {
  if (!ms3) return fail(EDTB200_EINVAL, "null pointer");
  ms3[0] = ms3[1] = ms3[2] = 0.0f;
  if (steps_back < 0 || steps_back >= kProfileRing || steps_back >= g_pass_seq)
    return fail(EDTB200_EINVAL, "no profiled transform %d steps back", steps_back);
  const int slot = (int)((g_pass_seq - 1 - steps_back) % kProfileRing);
  for (int i = 0; i < g_pass_marks[slot] && i < 3; ++i) {
    if (!g_pass_events[slot][i] || !g_pass_events[slot][i + 1]) break;
    CUDA_TRY(cudaEventSynchronize(g_pass_events[slot][i + 1]));
    CUDA_TRY(cudaEventElapsedTime(&ms3[i], g_pass_events[slot][i], g_pass_events[slot][i + 1]));
  }
  return 0;
}

int edtb200_release(void) {
  DeviceGuard restore_device;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess) { cudaGetLastError(); return 0; }
  for (int d = 0; d < count && d < kMaxDevices; ++d) {
    DeviceCache& dc = g_cache[d];
    std::lock_guard<std::mutex> host_call(dc.host_call);
    std::lock_guard<std::mutex> guard(dc.lock);
    if (!dc.probed) continue;
    cudaSetDevice(d);
    cudaDeviceSynchronize();
    for (auto& t : dc.tables) {
      if (t.data) cudaFree(t.data);
      if (t.ready) cudaEventDestroy(t.ready);
      for (auto& e : t.used) if (e) cudaEventDestroy(e);
      t = DeviceCache::Table();
    }
    if (dc.stream) { cudaStreamSynchronize(dc.stream); cudaStreamDestroy(dc.stream); }
    if (dc.labels) cudaFree(dc.labels);
    if (dc.dist) cudaFree(dc.dist);
    if (dc.labels2) cudaFree(dc.labels2);
    if (dc.dist2) cudaFree(dc.dist2);
    if (dc.stream_up) cudaStreamDestroy(dc.stream_up);
    if (dc.stream_down) cudaStreamDestroy(dc.stream_down);
    for (int i = 0; i < 2; ++i) {
      if (dc.ev_up[i]) cudaEventDestroy(dc.ev_up[i]);
      if (dc.ev_comp[i]) cudaEventDestroy(dc.ev_comp[i]);
      if (dc.ev_down[i]) cudaEventDestroy(dc.ev_down[i]);
    }
    dc.labels = dc.labels2 = nullptr; dc.dist = dc.dist2 = nullptr;
    dc.labels_bytes = dc.labels2_bytes = dc.dist_bytes = dc.dist2_bytes = 0;
    dc.stream = dc.stream_up = dc.stream_down = nullptr;
    for (int i = 0; i < 2; ++i) dc.ev_up[i] = dc.ev_comp[i] = dc.ev_down[i] = nullptr;
    // everything the stream-ordered scratch pool still holds goes back to the driver
    if (dc.pool) cudaMemPoolTrimTo(dc.pool, 0);
    for (int dir = 0; dir < 2; ++dir) {
      StageBuffers& sb = g_stage[dir][d];
      for (int i = 0; i < kStages; ++i) {
        if (sb.buf[i]) { cudaFreeHost(sb.buf[i]); sb.buf[i] = nullptr; }
        if (sb.ev[i]) { cudaEventDestroy(sb.ev[i]); sb.ev[i] = nullptr; }
      }
    }
    cudaGetLastError();
  }
  return 0;
}

}  // extern "C"
