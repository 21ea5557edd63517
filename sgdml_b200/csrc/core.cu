// Error plumbing, host/device staging and misc entry points of the sgdml_b200 C ABI.
#include "common.cuh"

#include <algorithm>
#include <map>
#include <mutex>

namespace sgdml {

static thread_local std::string g_last_error;

void set_last_error(const std::string& msg) { g_last_error = msg; }

int fail_cuda(cudaError_t e, const char* what, const char* file, int line) {
  char buf[512];
  snprintf(buf, sizeof(buf), "CUDA error %d (%s) in `%s` at %s:%d", (int)e, cudaGetErrorString(e), what, file, line);
  g_last_error = buf;
  // leave no sticky "last error" behind for the next call's launch checks
  cudaGetLastError();
  return -(int)e;
}

int fail_arg(const char* what) {
  g_last_error = std::string("invalid argument: requirement `") + what + "` violated";
  return SGDML_B200_ERR_ARG;
}

int require_device() {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    cudaGetLastError();
    g_last_error =
        "sgdml_b200: no CUDA device visible -- this engine has no CPU fallback (H100 / sm_90a required)";
    return SGDML_B200_ERR_NO_DEVICE;
  }
  return 0;
}

bool is_device_ptr(const void* p) {
  if (p == nullptr) return false;
  cudaPointerAttributes attr;
  cudaError_t e = cudaPointerGetAttributes(&attr, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
}

int read_int64s(const int64_t* src, size_t n, std::vector<int64_t>& out) {
  out.resize(n);
  if (is_device_ptr(src))
    SG_CUDA(cudaMemcpy(out.data(), src, sizeof(int64_t) * n, cudaMemcpyDeviceToHost));
  else
    std::copy(src, src + n, out.begin());
  return 0;
}

// ---- staging-buffer pool (see the comment on class Staged)
namespace {
struct PoolBuf {
  void* p;
  size_t cap;
  int dev;
};
struct StagePool {
  std::vector<PoolBuf> free_;
  size_t bytes = 0;
};
thread_local StagePool g_pool;
constexpr size_t POOL_MAX_BUF = (size_t)256 << 20;     // larger staging buffers are not kept
constexpr size_t POOL_MAX_TOTAL = (size_t)1024 << 20;  // per host thread
constexpr size_t POOL_MAX_COUNT = 32;

cudaError_t pool_get(size_t bytes, int dev, void** out, size_t* cap) {
  int best = -1;
  for (int i = 0; i < (int)g_pool.free_.size(); ++i) {
    const PoolBuf& b = g_pool.free_[(size_t)i];
    if (b.dev == dev && b.cap >= bytes && b.cap <= 2 * bytes + 4096 &&
        (best < 0 || b.cap < g_pool.free_[(size_t)best].cap))
      best = i;
  }
  if (best >= 0) {
    *out = g_pool.free_[(size_t)best].p;
    *cap = g_pool.free_[(size_t)best].cap;
    g_pool.bytes -= *cap;
    g_pool.free_.erase(g_pool.free_.begin() + best);
    return cudaSuccess;
  }
  *cap = bytes;
  return cudaMalloc(out, bytes);
}

void pool_put(void* p, size_t cap, int dev) {
  if (cap > POOL_MAX_BUF) {
    cudaFree(p);
    return;
  }
  while (!g_pool.free_.empty() && (g_pool.bytes + cap > POOL_MAX_TOTAL || g_pool.free_.size() >= POOL_MAX_COUNT)) {
    cudaFree(g_pool.free_.front().p);  // oldest first
    g_pool.bytes -= g_pool.free_.front().cap;
    g_pool.free_.erase(g_pool.free_.begin());
  }
  g_pool.free_.push_back(PoolBuf{p, cap, dev});
  g_pool.bytes += cap;
}
}  // namespace

Staged::~Staged() {
  if (owns_ && dev_) {
    cudaStreamSynchronize(stream_);  // nothing queued on the buffer's stream may still touch it
    pool_put(dev_, cap_, dev_id_);
  }
}

int Staged::init(const void* user, size_t bytes, bool copy_in, cudaStream_t s) {
  user_ = const_cast<void*>(user);
  bytes_ = bytes;
  stream_ = s;
  if (user == nullptr || bytes == 0) {
    dev_ = nullptr;
    owns_ = false;
    return 0;
  }
  if (is_device_ptr(user)) {
    dev_ = user_;
    owns_ = false;
    return 0;
  }
  SG_CUDA(cudaGetDevice(&dev_id_));
  SG_CUDA(pool_get(bytes, dev_id_, &dev_, &cap_));
  owns_ = true;
  if (copy_in) SG_CUDA(cudaMemcpyAsync(dev_, user, bytes, cudaMemcpyHostToDevice, s));
  return 0;
}

int Staged::finish(cudaStream_t s) {
  if (owns_ && dev_ && user_) SG_CUDA(cudaMemcpyAsync(user_, dev_, bytes_, cudaMemcpyDeviceToHost, s));
  return 0;
}

namespace {
struct WsBuf {
  void* p = nullptr;
  size_t cap = 0;
};
WsBuf g_ws[64][WS_SLOT_COUNT];
}  // namespace

int ws_get(int slot, size_t bytes, void** out) {
  int dev = 0;
  SG_CUDA(cudaGetDevice(&dev));
  SG_ARG(dev >= 0 && dev < 64 && slot >= 0 && slot < WS_SLOT_COUNT);
  WsBuf& b = g_ws[dev][slot];
  if (b.cap < bytes) {
    if (b.p != nullptr) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
    SG_CUDA(cudaMalloc(&b.p, bytes));
    b.cap = bytes;
  }
  *out = b.p;
  return 0;
}

namespace {
struct CacheKey {
  int dev;
  size_t bytes;
  bool operator<(const CacheKey& o) const { return dev != o.dev ? dev < o.dev : bytes < o.bytes; }
};
std::mutex g_cache_mu;
std::map<void*, CacheKey> g_cache_live;        // blocks handed out by cached_malloc
std::multimap<CacheKey, void*> g_cache_free;   // blocks kept for reuse
size_t g_cache_bytes = 0;
constexpr size_t CACHE_LIMIT_BYTES = 8ull << 30;
}  // namespace

void cache_release_all() {
  std::lock_guard<std::mutex> lk(g_cache_mu);
  for (auto& kv : g_cache_free) cudaFree(kv.second);
  g_cache_free.clear();
  g_cache_bytes = 0;
}

cudaError_t cached_malloc_bytes(void** p, size_t bytes) {
  *p = nullptr;
  if (bytes == 0) return cudaSuccess;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const CacheKey key{dev, bytes};
  {
    std::lock_guard<std::mutex> lk(g_cache_mu);
    auto it = g_cache_free.find(key);
    if (it != g_cache_free.end()) {
      *p = it->second;
      g_cache_free.erase(it);
      g_cache_bytes -= bytes;
      g_cache_live[*p] = key;
      return cudaSuccess;
    }
  }
  e = cudaMalloc(p, bytes);
  if (e == cudaErrorMemoryAllocation) {  // give the cached blocks back and try once more
    cudaGetLastError();
    cache_release_all();
    e = cudaMalloc(p, bytes);
  }
  if (e == cudaSuccess) {
    std::lock_guard<std::mutex> lk(g_cache_mu);
    g_cache_live[*p] = key;
  }
  return e;
}

cudaError_t cached_free(void* p) {
  if (p == nullptr) return cudaSuccess;
  {
    std::lock_guard<std::mutex> lk(g_cache_mu);
    auto it = g_cache_live.find(p);
    if (it != g_cache_live.end()) {
      const CacheKey key = it->second;
      g_cache_live.erase(it);
      if (g_cache_bytes + key.bytes <= CACHE_LIMIT_BYTES) {
        g_cache_free.emplace(key, p);
        g_cache_bytes += key.bytes;
        return cudaSuccess;
      }
    }
  }
  return cudaFree(p);
}

int num_sms() {
  static int cached[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev < 0 || dev >= 64) return 132;
  if (cached[dev] == 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cached[dev] = n;
  }
  return cached[dev];
}

// ---- launch accounting / profiling
static long long g_launches[KID_COUNT] = {0};
static double g_prof_ms[KID_COUNT] = {0};
static long long g_prof_n[KID_COUNT] = {0};
static int g_prof_enabled = 0;

void count_launch(int kid, int n) {
  if (kid >= 0 && kid < KID_COUNT) g_launches[kid] += n;
}
bool profiling_enabled() { return g_prof_enabled != 0; }

ProfScope::ProfScope(int kid, cudaStream_t s) : kid_(kid), s_(s) {
  if (!g_prof_enabled) return;
  if (cudaEventCreate(&e0_) != cudaSuccess || cudaEventCreate(&e1_) != cudaSuccess) {
    e0_ = e1_ = nullptr;
    return;
  }
  cudaEventRecord(e0_, s_);
}
ProfScope::~ProfScope() {
  if (e0_ == nullptr || e1_ == nullptr) return;
  cudaEventRecord(e1_, s_);
  if (cudaEventSynchronize(e1_) == cudaSuccess) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, e0_, e1_) == cudaSuccess) {
      g_prof_ms[kid_] += ms;
      g_prof_n[kid_] += 1;
    }
  }
  cudaEventDestroy(e0_);
  cudaEventDestroy(e1_);
}

}  // namespace sgdml

extern "C" {

int sgdml_b200_profile_enable(int on) {
  sgdml::g_prof_enabled = on;
  return 0;
}
int sgdml_b200_profile_reset(void) {
  for (int i = 0; i < sgdml::KID_COUNT; ++i) {
    sgdml::g_prof_ms[i] = 0;
    sgdml::g_prof_n[i] = 0;
    sgdml::g_launches[i] = 0;
  }
  return 0;
}
int sgdml_b200_profile_get(int kid, double* total_ms, int64_t* scopes, int64_t* launches) {
  if (kid < 0 || kid >= sgdml::KID_COUNT) return SGDML_B200_ERR_ARG;
  if (total_ms) *total_ms = sgdml::g_prof_ms[kid];
  if (scopes) *scopes = sgdml::g_prof_n[kid];
  if (launches) *launches = sgdml::g_launches[kid];
  return 0;
}

int sgdml_b200_release_workspaces(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
  cudaDeviceSynchronize();
  for (int i = 0; i < sgdml::WS_SLOT_COUNT; ++i) {
    if (sgdml::g_ws[dev][i].p != nullptr) cudaFree(sgdml::g_ws[dev][i].p);
    sgdml::g_ws[dev][i] = sgdml::WsBuf();
  }
  sgdml::cache_release_all();
  return 0;
}

int sgdml_b200_abi_version(void) { return SGDML_B200_ABI_VERSION; }

const char* sgdml_b200_last_error(void) { return sgdml::g_last_error.c_str(); }

int sgdml_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

}  // extern "C"
