/* TEST INFRASTRUCTURE ONLY (oracle shim) - the <volk/volk.h> that pulse_blanking_cc.cc sees (oracle/filter.mk puts this
 * directory ahead of oracle/shim): the shim's kernels, plus the one more the blanker calls. */
#pragma once
#include_next <volk/volk.h>
/* pulse_blanking_cc.cc:75: the generic kernel, an ascending sum from 0.0 with every addition rounded on its own
 * (-ffp-contract=off and no -ffast-math keep the compiler from reordering it) */
static inline void volk_32f_accumulator_s32f(float* result, const float* in, unsigned int n)
{
    float r = 0.f;
    for (unsigned int i = 0; i < n; i++) r += in[i];
    *result = r;
}
