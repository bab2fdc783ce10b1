// Error reporting, version, device probe.
#include <stdarg.h>

#include <mutex>
#include <vector>

#include "common.cuh"

namespace gantts {
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) in %s", static_cast<int>(e), cudaGetErrorString(e), what);
  return GANTTS_E_CUDA;
}

static long long g_launches = 0;
void count_launch() { ++g_launches; }

struct ProfRec {
  cudaEvent_t e0, e1;
  int kind;
  double work;
};
static bool g_prof_on = false;
static std::vector<ProfRec> g_recs;
static std::vector<cudaEvent_t> g_pool;
static ProfRec g_open;
static bool g_open_valid = false;

static cudaEvent_t get_event() {
  cudaEvent_t e;
  if (!g_pool.empty()) {
    e = g_pool.back();
    g_pool.pop_back();
    return e;
  }
  cudaEventCreate(&e);
  return e;
}

void prof_begin(int kind, double work, cudaStream_t st) {
  if (!g_prof_on) return;
  g_open.e0 = get_event();
  g_open.e1 = get_event();
  g_open.kind = kind;
  g_open.work = work;
  cudaEventRecord(g_open.e0, st);
  g_open_valid = true;
}

void prof_end(cudaStream_t st) {
  if (!g_prof_on || !g_open_valid) return;
  cudaEventRecord(g_open.e1, st);
  g_recs.push_back(g_open);
  g_open_valid = false;
}

// The side and branch streams of each device (created on first use) and the one event that orders them against the
// caller's stream.
// stream_wait records and waits under one lock, so no other thread can re-record the event between the two calls.
struct SideStream {
  cudaStream_t st = nullptr;
  cudaStream_t branch = nullptr;
  cudaEvent_t ev = nullptr;
};
static std::mutex g_side_mu;
static SideStream g_side[64];

static int side_locked(SideStream** out) {
  int dev = 0;
  GANTTS_CUDA(cudaGetDevice(&dev));
  GANTTS_CHECK_ARG(dev >= 0 && dev < 64, "side stream: device ordinal %d out of range", dev);
  SideStream& s = g_side[dev];
  if (!s.ev) GANTTS_CUDA(cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming));
  if (!s.st) {
    // the device's highest priority: when a running GEMM's last wave frees SMs, the block scheduler dispatches the side
    // branch's waiting blocks before those of the next GEMM the caller's stream launched early under PDL, so the two
    // chains alternate and each fills the other's tail instead of the whole input-gradient chain running first
    int least = 0, greatest = 0;
    GANTTS_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    GANTTS_CUDA(cudaStreamCreateWithPriority(&s.st, cudaStreamNonBlocking, greatest));
  }
  if (!s.branch) {
    // the device's lowest priority (a caller's default stream has it too): at the highest, the branch's GEMMs took the
    // SMs the generator forward's GEMMs were waiting for and the cfg2 step got slower (DESIGN.md section 5)
    int least = 0, greatest = 0;
    GANTTS_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
    GANTTS_CUDA(cudaStreamCreateWithPriority(&s.branch, cudaStreamNonBlocking, least));
  }
  *out = &s;
  return GANTTS_OK;
}

int side_stream(cudaStream_t* out) {
  std::lock_guard<std::mutex> lk(g_side_mu);
  SideStream* s;
  int rc = side_locked(&s);
  if (rc) return rc;
  *out = s->st;
  return GANTTS_OK;
}

int branch_stream(cudaStream_t* out) {
  std::lock_guard<std::mutex> lk(g_side_mu);
  SideStream* s;
  int rc = side_locked(&s);
  if (rc) return rc;
  *out = s->branch;
  return GANTTS_OK;
}

int stream_wait(cudaStream_t waiter, cudaStream_t on) {
  std::lock_guard<std::mutex> lk(g_side_mu);
  SideStream* s;
  int rc = side_locked(&s);
  if (rc) return rc;
  GANTTS_CUDA(cudaEventRecord(s->ev, on));
  GANTTS_CUDA(cudaStreamWaitEvent(waiter, s->ev, 0));
  return GANTTS_OK;
}
}  // namespace gantts

extern "C" long long gantts_launch_count(void) { return gantts::g_launches; }

extern "C" int gantts_profile_enable(int on) {
  gantts::g_prof_on = on != 0;
  return GANTTS_OK;
}

// Synchronises the recorded events, ADDS per-kind totals into the caller's arrays (length 8 each:
// milliseconds, work units, launches) and recycles the events.
extern "C" int gantts_profile_collect(double* ms, double* work, long long* launches) {
  using namespace gantts;
  for (auto& r : g_recs) {
    float t = 0.f;
    cudaError_t e = cudaEventSynchronize(r.e1);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&t, r.e0, r.e1);
    if (e != cudaSuccess) return cuda_fail(e, "profile_collect");
    if (r.kind >= 0 && r.kind < PROF_KINDS) {
      if (ms) ms[r.kind] += t;
      if (work) work[r.kind] += r.work;
      if (launches) launches[r.kind] += 1;
    }
    g_pool.push_back(r.e0);
    g_pool.push_back(r.e1);
  }
  g_recs.clear();
  return GANTTS_OK;
}

extern "C" int gantts_version(void) { return 104; }

extern "C" const char* gantts_last_error_string(void) { return gantts::g_err; }

extern "C" int gantts_device_supported(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return 0;
  return (prop.major == 9 && prop.minor == 0) ? 1 : 0;
}
