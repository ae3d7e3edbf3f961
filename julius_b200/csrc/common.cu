// common.cu -- error string, launch counter, version, addlog table.
#include "common.cuh"
#include <cstdarg>
#include <cmath>

namespace jb200 {
static thread_local char g_err[1024] = "";
std::atomic<int64_t> g_launches{0};

void build_addlog_table(std::vector<float> &tbl) {
  tbl.resize(ADDLOG_TABLE_N);
  for (int i = 0; i < ADDLOG_TABLE_N; i++) {
    float f = -((float)15 * (float)i / (float)ADDLOG_TABLE_N);
    tbl[i] = (float)log(1 + exp((double)f));
  }
}

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace jb200

extern "C" int jb200_version(void) { return 100; }
extern "C" const char *jb200_last_error(void) { return jb200::g_err; }
extern "C" int64_t jb200_launch_count(void) { return jb200::g_launches.load(); }
extern "C" int jb200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}
