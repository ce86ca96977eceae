#include "common.cuh"

#include <cstdarg>
#include <mutex>
#include <string>
#include <vector>

namespace tapir {

namespace {
thread_local char g_error[1024] = "";
}

unsigned long long g_launch_count = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

const char* last_error() { return g_error; }

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return kCudaError;
}

// ------------------------------------------------------------------------ profiling
bool g_profile_on = false;
namespace {
struct ProfRec {
  cudaEvent_t a, b;
  int name_id;
  double flops, bytes;
};
std::vector<ProfRec> g_recs;
std::vector<std::string> g_names;
std::vector<cudaEvent_t> g_event_pool;  // events are recycled: creating them in the launch
                                        // path starves the GPU and inflates the timings
bool take_event(cudaEvent_t* e) {
  if (g_event_pool.empty()) {
    for (int i = 0; i < 1024; ++i) {
      cudaEvent_t ev;
      if (cudaEventCreate(&ev) != cudaSuccess) break;
      g_event_pool.push_back(ev);
    }
    if (g_event_pool.empty()) return false;
  }
  *e = g_event_pool.back();
  g_event_pool.pop_back();
  return true;
}
int name_id(const char* n) {
  for (size_t i = 0; i < g_names.size(); ++i)
    if (g_names[i] == n) return (int)i;
  g_names.emplace_back(n);
  return (int)g_names.size() - 1;
}
}  // namespace

ProfileScope::ProfileScope(const char* name, cudaStream_t s, double flops, double bytes)
    : slot(-1), stream(s) {
  if (!g_profile_on) return;
  ProfRec r;
  if (!take_event(&r.a) || !take_event(&r.b)) return;
  r.name_id = name_id(name);
  r.flops = flops;
  r.bytes = bytes;
  cudaEventRecord(r.a, s);
  g_recs.push_back(r);
  slot = (int)g_recs.size() - 1;
}
ProfileScope::~ProfileScope() {
  if (slot >= 0) cudaEventRecord(g_recs[slot].b, stream);
}

void profile_enable(int on) {
  g_profile_on = on != 0;
  if (g_profile_on && g_event_pool.size() < 2048) {  // pre-create outside the timed launches
    for (int i = 0; i < 2048; ++i) {
      cudaEvent_t ev;
      if (cudaEventCreate(&ev) != cudaSuccess) break;
      g_event_pool.push_back(ev);
    }
  }
}

// Synchronises, aggregates per name and clears.  JSON: {"name": {"launches":n,"ms":t,
// "flops":f,"bytes":b}, ...}
int profile_report(char* buf, size_t cap) {
  cudaDeviceSynchronize();
  struct Agg { long long n = 0; double ms = 0, flops = 0, bytes = 0; };
  std::vector<Agg> agg(g_names.size());
  for (auto& r : g_recs) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
      Agg& a = agg[r.name_id];
      a.n += 1; a.ms += ms; a.flops += r.flops; a.bytes += r.bytes;
    }
    g_event_pool.push_back(r.a);
    g_event_pool.push_back(r.b);
  }
  g_recs.clear();
  std::string out = "{";
  bool first = true;
  for (size_t i = 0; i < g_names.size(); ++i) {
    if (agg[i].n == 0) continue;
    char line[512];
    snprintf(line, sizeof(line), "%s\"%s\": {\"launches\": %lld, \"ms\": %.6f, \"flops\": %.6e, \"bytes\": %.6e}",
             first ? "" : ", ", g_names[i].c_str(), agg[i].n, agg[i].ms, agg[i].flops, agg[i].bytes);
    out += line;
    first = false;
  }
  out += "}";
  if (out.size() + 1 > cap) {
    set_error("profile_report: buffer too small (%zu needed)", out.size() + 1);
    return kBadArgument;
  }
  memcpy(buf, out.c_str(), out.size() + 1);
  return kOk;
}

int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) dev = 0;
  return dev < kMaxDevices ? dev : kMaxDevices - 1;
}

int num_sms() {
  static int n[kMaxDevices] = {};
  const int dev = current_device();
  if (n[dev] == 0) {
    if (cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n[dev] <= 0)
      n[dev] = 132;
  }
  return n[dev];
}

}  // namespace tapir
