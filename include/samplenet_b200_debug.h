/* samplenet_b200_debug.h -- bring-up instrumentation of libsamplenet_b200.so.  NOT part of the drop-in surface (include/samplenet_b200.h):
 * one tensor-core GEMM tile with overridable descriptor encodings, and clock64 timelines of the fused kernels.  Used by tools/ and tests only. */
#ifndef SAMPLENET_B200_DEBUG_H
#define SAMPLENET_B200_DEBUG_H
#include "samplenet_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Bring-up / unit-test hook of the wgmma layer kernel (csrc/encoder_tc.cu): D (rows, c_out) = A (rows, c_in) * W (c_out, c_in)^T + bias
 * as 3xTF32 on the tensor cores.  desc_hi / k_adv16 / swizzle override the shared-memory descriptor encoding (0,0,0 = defaults);
 * they exist so that one GPU session can sweep encodings.  c_in % 8 == 0, 8 <= c_in, c_out <= 256. */
int snb200_debug_tc_gemm(int rows, int c_in, int c_out, const float *A, const float *W, const float *bias, float *D,
                         unsigned desc_hi, int k_adv16, int swizzle, snb200_stream_t stream);

/* Bring-up instrumentation: 64 SM-clock timestamps written by CTA 0 of the last FC-head launch (synchronous copy). */
int snb200_debug_head_timestamps(long long *host_out64);
int snb200_debug_conv_stack_timestamps(long long *host_out64);

#ifdef __cplusplus
}
#endif
#endif
