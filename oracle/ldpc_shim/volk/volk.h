/*
 * TEST INFRASTRUCTURE ONLY (oracle, LDPC part). The VOLK stand-in of oracle/shim plus the two entry points the CCSDS LDPC
 * decoder's translation units call: the convert kernel without the _u suffix (generic_correlator.cpp:178), the same generic
 * divide-by-scalar loop, and volk_get_machine() (cpu_features.cpp:9), which names no SIMD extension, so that
 * get_best_ldpc_decoder (ldpc_decoder.cpp:20-36) picks the generic decoder by its own logic.
 */
#pragma once
#include "../../shim/volk/volk.h"
#ifdef __cplusplus
extern "C" {
#endif
static inline void volk_8i_s32f_convert_32f(float *out, const int8_t *in, const float scalar, unsigned int num_points)
{
    volk_8i_s32f_convert_32f_u(out, in, scalar, num_points);
}
static inline const char *volk_get_machine(void) { return "generic"; }
#ifdef __cplusplus
}
#endif
