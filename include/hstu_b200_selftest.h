/*
 * hstu_b200_selftest.h -- C ABI of libhstu_b200_selftest.so: TEST INFRASTRUCTURE, not part of the product library.
 *
 * On-device self test of the sm_90a primitives the attention kernels of libhstu_b200.so are built from (TMA loads of
 * swizzled boxes, wgmma with K-major and MN-major shared-memory operands and with A from registers).  Built from
 * csrc/wgmma_selftest.cu + csrc/tmap.cu by generative_recommenders_b200/build.py.  The entry point keeps its earlier name.
 */
#ifndef HSTU_B200_SELFTEST_H_
#define HSTU_B200_SELFTEST_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Writes a report into `report` (host buffer).  Returns the number of failed checks (0 = all good, <0 = could not run). */
int hstu_umma_selftest(char* report, size_t report_bytes);
const char* hstu_selftest_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* HSTU_B200_SELFTEST_H_ */
