// capi.cu — error reporting and device queries of the C ABI (include/lkpy_b200.h).

#include <cstdarg>
#include <cstdlib>

#include "common.cuh"

namespace lk {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

// ---------------------------------------------------------------------------
// Diagnostic switches.  The LK_* environment variables are read ONCE, when the first
// entry point that needs them runs (never per launch); lk_set_option changes a
// switch afterwards (tests and tools/ use it to reach the non-default kernels).
// ---------------------------------------------------------------------------
struct OptionDef {
    const char *name;  // also the environment variable
    int Options::*field;
};
static const OptionDef OPTION_DEFS[] = {
    {"LK_ALS_TC", &Options::als_tc},
    {"LK_ALS_TF32", &Options::als_tf32},
    {"LK_KNN_WARPS", &Options::knn_warps},
    {"LK_KNN_CTAS", &Options::knn_ctas},
    {"LK_KNN_SCORE_CTAS", &Options::knn_score_ctas},
};

Options &options()
{
    static Options o = [] {
        Options v;
        for (const OptionDef &d : OPTION_DEFS)
            if (const char *e = getenv(d.name))
                if (e[0] != '\0') v.*(d.field) = atoi(e);
        return v;
    }();
    return o;
}

int sm_count()
{
    static int cached = 0;
    if (cached == 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) == cudaSuccess &&
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
            cached = n;
        else
            return 132;  // H100 SXM
    }
    return cached;
}

}  // namespace lk

extern "C" {

int lk_version(void) { return 114; }

const char *lk_last_error(void) { return lk::g_err; }

int lk_set_option(const char *name, int value)
{
    LK_REQUIRE(name != nullptr, LK_ERR_INVALID, "lk_set_option: null name");
    for (const lk::OptionDef &d : lk::OPTION_DEFS)
        if (strcmp(d.name, name) == 0) {
            lk::options().*(d.field) = value;
            return LK_OK;
        }
    lk::set_error("lk_set_option: unknown option %s", name);
    return LK_ERR_INVALID;
}

int lk_get_option(const char *name, int *value)
{
    LK_REQUIRE(name != nullptr && value != nullptr, LK_ERR_INVALID, "lk_get_option: null argument");
    for (const lk::OptionDef &d : lk::OPTION_DEFS)
        if (strcmp(d.name, name) == 0) {
            *value = lk::options().*(d.field);
            return LK_OK;
        }
    lk::set_error("lk_get_option: unknown option %s", name);
    return LK_ERR_INVALID;
}

int lk_device_info(int *sm_count, int *cc)
{
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) {
        lk::set_error("no CUDA device: %s", cudaGetErrorString(e));
        return LK_ERR_NO_DEVICE;
    }
    int n = 0, major = 0, minor = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
    if (sm_count) *sm_count = n;
    if (cc) *cc = major * 10 + minor;
    return LK_OK;
}

}  // extern "C"
