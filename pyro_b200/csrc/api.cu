// api.cu -- error strings, version, launch counter.
#include "b2_common.cuh"

namespace b2 {
int64_t g_launch_count = 0;
}

extern "C" const char* b2_last_error(int code) {
  switch (code) {
    case B2_OK: return "ok";
    case B2_ERR_BAD_DTYPE: return "unsupported or inconsistent dtype";
    case B2_ERR_BAD_SHAPE: return "bad shape / ndim / stride";
    case B2_ERR_BAD_FAMILY: return "unknown distribution family or model id";
    case B2_ERR_NULL: return "required pointer is null";
    case B2_ERR_WORKSPACE: return "workspace missing or too small";
    case B2_ERR_UNSUPPORTED_REDUCTION: return "gradient output broadcast pattern is not fused";
    case B2_ERR_LAUNCH: return "CUDA kernel launch failed";
    case B2_ERR_TOO_LARGE: return "problem size exceeds the limits of this entry point";
    case B2_ERR_NO_DEVICE: return "no CUDA device";
    default: return "unknown error";
  }
}

extern "C" int b2_version(void) { return 104; }
extern "C" int64_t b2_launch_count(void) { return b2::g_launch_count; }
