// cabi.cu -- library-level entry points of include/scn_kernels.h: version, launch counter and
// the optional per-kernel event timing used by bench.py's roofline leg.
#include <stdio.h>
#include <string.h>

#include <map>
#include <mutex>
#include <set>
#include <string>
#include <vector>

#include "scn_common.cuh"

namespace scn {
std::atomic<uint64_t> g_launches{0};
std::atomic<int> g_prof_on{0};

namespace {
struct Rec {
  const char* name;
  cudaEvent_t a, b;
};
std::mutex g_prof_mu;
std::vector<Rec*> g_recs;
}  // namespace

void prof_begin(const char* name, cudaStream_t st, void** token) {
  Rec* r = new Rec{name, nullptr, nullptr};
  if (cudaEventCreate(&r->a) != cudaSuccess || cudaEventCreate(&r->b) != cudaSuccess) {
    delete r;
    return;
  }
  cudaEventRecord(r->a, st);
  *token = r;
}

void prof_end(void* token, cudaStream_t st) {
  Rec* r = static_cast<Rec*>(token);
  cudaEventRecord(r->b, st);
  std::lock_guard<std::mutex> g(g_prof_mu);
  g_recs.push_back(r);
}

int raise_smem_limit(const void* kernel, size_t bytes) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;  // (kernel, device) pairs already raised
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) {
    std::lock_guard<std::mutex> g(mu);
    if (done.count({kernel, dev})) return 0;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) {
      done.insert({kernel, dev});
      return 0;
    }
  }
  cudaGetLastError();  // reported here, so that later calls report their own errors
  return (int)e;
}

}  // namespace scn

extern "C" int scn_abi_version(void) { return 1; }
extern "C" uint64_t scn_launch_count(void) {
  return scn::g_launches.load(std::memory_order_relaxed);
}

extern "C" void scn_prof_enable(int on) {
  using namespace scn;
  if (on) {
    std::lock_guard<std::mutex> g(g_prof_mu);
    for (Rec* r : g_recs) {
      cudaEventDestroy(r->a);
      cudaEventDestroy(r->b);
      delete r;
    }
    g_recs.clear();
  }
  g_prof_on.store(on ? 1 : 0);
}

extern "C" int scn_prof_report(char* host_buf, size_t cap) {
  using namespace scn;
  if (!host_buf || cap < 4) return SCN_E_BADARG;
  std::map<std::string, std::pair<uint64_t, double>> agg;
  {
    std::lock_guard<std::mutex> g(g_prof_mu);
    for (Rec* r : g_recs) {
      if (cudaEventSynchronize(r->b) != cudaSuccess) return -100;
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, r->a, r->b) != cudaSuccess) return -101;
      auto& e = agg[r->name];
      e.first += 1;
      e.second += ms;
    }
  }
  if (agg.empty()) {
    host_buf[0] = 0;
    return 0;
  }
  std::string s = "{";
  bool first = true;
  for (auto& kv : agg) {
    char tmp[256];
    snprintf(tmp, sizeof(tmp), "%s\"%s\": {\"launches\": %llu, \"ms\": %.6f}", first ? "" : ", ",
             kv.first.c_str(), (unsigned long long)kv.second.first, kv.second.second);
    s += tmp;
    first = false;
  }
  s += "}";
  if (s.size() + 1 > cap) return SCN_E_BADARG;
  memcpy(host_buf, s.c_str(), s.size() + 1);
  return (int)s.size();
}
