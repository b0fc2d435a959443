// the one translation unit of libdfx_emu_full.so that defines the context-switch primitive of simt.h,
// and the launch log of DFX_LAUNCH (dfx_common.cuh, DFX_EMU branch)
#define SIMT_IMPLEMENTATION
#include <cuda_runtime.h>

#include <cxxabi.h>
#include <dlfcn.h>

#include <mutex>
#include <string>
#include <vector>

static std::mutex g_log_mu;
static std::vector<const void*> g_log;  // launched kernels, in launch order

void dfx_emu_record_launch(const void* kernel) {
    std::lock_guard<std::mutex> lk(g_log_mu);
    g_log.push_back(kernel);
}

static std::string kernel_name(const void* kernel) {
    Dl_info info;
    if (!dladdr(kernel, &info) || !info.dli_sname || info.dli_saddr != kernel) return "?";
    int status = 0;
    char* dem = abi::__cxa_demangle(info.dli_sname, nullptr, nullptr, &status);
    std::string out = (status == 0 && dem) ? dem : info.dli_sname;
    free(dem);
    return out;
}

// The demangled names of the kernels launched since the last call, one per line, into buf.  Returns
// the bytes the names take with the terminating NUL; the log is cleared only when they fit in cap
// (call with cap = 0 to size the buffer).  A kernel that is not an exported symbol shows as "?".
extern "C" int64_t dfx_emu_launch_log(char* buf, int64_t cap) {
    std::lock_guard<std::mutex> lk(g_log_mu);
    std::string all;
    for (const void* k : g_log) all += kernel_name(k) + "\n";
    const int64_t need = (int64_t)all.size() + 1;
    if (buf && cap >= need) {
        memcpy(buf, all.c_str(), (size_t)need);
        g_log.clear();
    }
    return need;
}
