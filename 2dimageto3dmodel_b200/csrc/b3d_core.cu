// libb3d core: thread-local error string, version, launch counter, kernel-variant record.
#include <atomic>
#include <stdarg.h>
#include <string.h>

#include "b3d_common.cuh"

namespace b3d {
static thread_local char g_err[512] = "";
static thread_local char g_variant[256] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void clear_variant() { g_variant[0] = 0; }
void add_variant(const char* fmt, ...) {
    size_t n = strlen(g_variant);
    if (n + 2 >= sizeof(g_variant)) return;
    if (n) g_variant[n++] = ';';
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_variant + n, sizeof(g_variant) - n, fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }
}  // namespace b3d

extern "C" {
const char* b3d_last_error(void) { return b3d::g_err; }
const char* b3d_last_variant(void) { return b3d::g_variant; }
int b3d_version(void) { return 410; }   // 4.1: b3d_sample_pack (sample export)
uint64_t b3d_launch_count(void) { return b3d::g_launches.load(std::memory_order_relaxed); }
}
