/* TEST INFRASTRUCTURE ONLY (oracle shim) - the <volk/volk.h> that notch_cc.cc and notch_lite_cc.cc see (oracle/notch.mk puts
 * this directory ahead of oracle/shim_input_filter and oracle/shim): those shims' kernels, plus the five more the notch
 * filters call.  Each one restates the generic protokernel of VOLK 2.5 (LV_HAVE_GENERIC); VOLK is not installed here.  An
 * AVX-dispatched VOLK may differ from these in the last bit.  -ffp-contract=off keeps every product and sum rounded on its
 * own. */
#pragma once
#include_next <volk/volk.h>
#include <cmath>

/* 10 log10 of |x|^2 / normalizationFactor^2, the 1e-20 guarding log10 of 0 */
static inline void volk_32fc_s32f_power_spectrum_32f(float* logPowerOutput, const lv_32fc_t* complexFFTInput, const float normalizationFactor,
    unsigned int num_points)
{
    const float* inputPtr = reinterpret_cast<const float*>(complexFFTInput);
    const float iNormalizationFactor = 1.0 / normalizationFactor;
    for (unsigned int number = 0; number < num_points; number++)
        {
            const float real = *inputPtr++ * iNormalizationFactor;
            const float imag = *inputPtr++ * iNormalizationFactor;
            *logPowerOutput++ = 10.0 * log10f(((real * real) + (imag * imag)) + 1e-20);
        }
}

/* the mean of the bins at most spectralExclusionValue above the mean of all bins (the mean plus the exclusion if none) */
static inline void volk_32f_s32f_calc_spectral_noise_floor_32f(float* noiseFloorAmplitude, const float* realDataPoints,
    const float spectralExclusionValue, const unsigned int num_points)
{
    float sumMean = 0.0;
    for (unsigned int number = 0; number < num_points; number++) sumMean += realDataPoints[number];
    const float meanAmplitude = (sumMean / num_points) + spectralExclusionValue;
    sumMean = 0.0;
    unsigned int newNumDataPoints = num_points;
    for (unsigned int number = 0; number < num_points; number++)
        {
            if (realDataPoints[number] <= meanAmplitude)
                sumMean += realDataPoints[number];
            else
                newNumDataPoints--;
        }
    float localNoiseFloorAmplitude = 0;
    if (newNumDataPoints == 0)
        localNoiseFloorAmplitude = meanAmplitude;
    else
        localNoiseFloorAmplitude = sumMean / ((float)newNumDataPoints);
    *noiseFloorAmplitude = localNoiseFloorAmplitude;
}

/* sum of input[i] conj(taps[i]): even and odd items into two sums, added, then the last item when num_points is odd */
static inline void volk_32fc_x2_conjugate_dot_prod_32fc(lv_32fc_t* result, const lv_32fc_t* input, const lv_32fc_t* taps,
    unsigned int num_points)
{
    const unsigned int num_bytes = num_points * 8;
    float* res = reinterpret_cast<float*>(result);
    const float* in = reinterpret_cast<const float*>(input);
    const float* tp = reinterpret_cast<const float*>(taps);
    const unsigned int n_2_ccomplex_blocks = num_bytes >> 4;
    float sum0[2] = {0, 0};
    float sum1[2] = {0, 0};
    for (unsigned int i = 0; i < n_2_ccomplex_blocks; ++i)
        {
            sum0[0] += in[0] * tp[0] + in[1] * tp[1];
            sum0[1] += (-in[0] * tp[1]) + in[1] * tp[0];
            sum1[0] += in[2] * tp[2] + in[3] * tp[3];
            sum1[1] += (-in[2] * tp[3]) + in[3] * tp[2];
            in += 4;
            tp += 4;
        }
    res[0] = sum0[0] + sum1[0];
    res[1] = sum0[1] + sum1[1];
    if (num_bytes >> 3 & 1) *result += input[(num_bytes >> 3) - 1] * lv_conj(taps[(num_bytes >> 3) - 1]);
}

/* c[i] = a[i] conj(b[i]) */
static inline void volk_32fc_x2_multiply_conjugate_32fc(lv_32fc_t* cVector, const lv_32fc_t* aVector, const lv_32fc_t* bVector,
    unsigned int num_points)
{
    for (unsigned int number = 0; number < num_points; number++) cVector[number] = aVector[number] * lv_conj(bVector[number]);
}

/* atan2f(im, re) / normalizeFactor */
static inline void volk_32fc_s32f_atan2_32f(float* outputVector, const lv_32fc_t* inputVector, const float normalizeFactor,
    unsigned int num_points)
{
    const float* inPtr = reinterpret_cast<const float*>(inputVector);
    const float invNormalizeFactor = 1.0 / normalizeFactor;
    for (unsigned int number = 0; number < num_points; number++)
        {
            const float real = *inPtr++;
            const float imag = *inPtr++;
            outputVector[number] = atan2f(imag, real) * invNormalizeFactor;
        }
}
