// Error channel, version and launch counter of the neuralsim_b200 C ABI.
#include <stdarg.h>

#include <map>
#include <mutex>
#include <tuple>
#include <utility>

#include "nsb_common.cuh"

namespace nsb {
static thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
}  // namespace nsb

namespace nsb { std::atomic<int> g_opt_sdf_simt{0}; }

namespace nsb {
static thread_local DevCounts g_counts{nullptr, nullptr};
DevCounts take_counts() {
    const DevCounts c = g_counts;
    g_counts = DevCounts{nullptr, nullptr};
    return c;
}

static thread_local const int32_t *g_max_level = nullptr;
const int32_t *take_max_level() {
    const int32_t *l = g_max_level;
    g_max_level = nullptr;
    return l;
}
}  // namespace nsb

namespace nsb {
bool smem_opt_in_needed(const void *kernel, int dev, int bytes) {
    static std::mutex mu;
    static std::map<std::pair<const void *, int>, int> granted;
    std::lock_guard<std::mutex> lock(mu);
    int &g = granted[std::make_pair(kernel, dev)];
    if (g >= bytes) return false;
    g = bytes;
    return true;
}

int max_active_ctas(const void *kernel, int dev, int block, int smem_bytes) {
    static std::mutex mu;
    static std::map<std::tuple<const void *, int, int, int>, int> known;
    const auto key = std::make_tuple(kernel, dev, block, smem_bytes);
    {
        std::lock_guard<std::mutex> lock(mu);
        const auto it = known.find(key);
        if (it != known.end()) return it->second;
    }
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, block, (size_t)smem_bytes) != cudaSuccess) {
        cudaGetLastError();
        return 0;                  // not cached: the caller reports it, and a later call asks again
    }
    std::lock_guard<std::mutex> lock(mu);
    known[key] = n;
    return n;
}
}  // namespace nsb

// See include/neuralsim_b200.h: the binding is consumed (and cleared) by the next count-aware launch of this thread.
extern "C" int nsb_bind_device_counts(const int64_t *count0, const int64_t *count1) {
    nsb::g_counts = nsb::DevCounts{count0, count1};
    return 0;
}

// See include/neuralsim_b200.h: consumed (and cleared) by the next level-aware launch of this thread.
extern "C" int nsb_bind_device_max_level(const int32_t *level) {
    nsb::g_max_level = level;
    return 0;
}

// Self-check switch.  "sdf_simt" = 1 routes nsb_fused_sdf* through the CUDA-core reference kernel of csrc/fused.cu instead of
// the wgmma kernel (used by the tests to cross-check the two).
extern "C" int nsb_set_option(const char *key, int value) {
    if (key && !strcmp(key, "sdf_simt")) { nsb::g_opt_sdf_simt.store(value); return 0; }
    nsb::set_error("nsb_set_option: unknown key '%s'", key ? key : "(null)");
    return 2;
}

extern "C" const char *nsb_last_error(void) { return nsb::g_err; }
extern "C" int nsb_version(void) { return 100; }
extern "C" uint64_t nsb_launch_count(void) { return nsb::g_launches.load(); }
