// Error plumbing of the C ABI: every entry point returns 0 on success, non-zero otherwise; the
// message of the most recent failure on the calling thread is available through dv3_last_error().
#include "common.cuh"
#include <stdarg.h>
#include <stdlib.h>

namespace dv3 {
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

const Config& config() {
    static const Config c = [] {
        Config v;
        const char* e = getenv("DV3_PDL");
        v.pdl = (e && atoi(e) == 0) ? 0 : 1;
        int dev = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        v.sms = sms > 0 ? sms : 132;
        // relative loss of the main accumulator (fp16 x fp16 products) per MMA, in units of 2^-25: 0.56 measured on an
        // H100 SXM with tools/trunc_bias.py
        e = getenv("DV3_TC_GAMMA");               // override, in units of 2^-25 per MMA
        v.tc_gamma = (e ? (float)atof(e) : 0.56f) * 2.98023224e-8f;
        return v;
    }();
    return c;
}

static unsigned long long g_launches = 0;
unsigned long long launch_count() { return g_launches; }

int check_launch(const char* what) {
    __atomic_add_fetch(&g_launches, 1ULL, __ATOMIC_RELAXED);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return 0;
    set_error("%s: %s", what, cudaGetErrorString(e));
    return (int)e;
}
}  // namespace dv3

extern "C" {
const char* dv3_last_error(void) { return dv3::g_err; }
int dv3_abi_version(void) { return 2; }
long long dv3_launch_count(void) { return (long long)dv3::launch_count(); }
}
