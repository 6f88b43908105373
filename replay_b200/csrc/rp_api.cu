// rp_api.cu - library-level entry points of the C ABI (include/rp_b200.h).
#include "rp_host.h"

RP_API const char* rp_version(void) { return "rp_b200 0.1 sm_90a"; }
