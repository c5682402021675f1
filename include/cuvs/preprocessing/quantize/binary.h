/*
 * Binary quantizer C boundary: float rows to packed bits, one bit per column.
 * Same ABI as the reference's c/include/cuvs/preprocessing/quantize/binary.h
 * (threshold enum, params struct, quantizer handle, Create/Destroy family,
 * Train, Transform, TransformWithParams).
 *
 * Bit j % 8 of byte j / 8 of an output row is set when column j exceeds its
 * threshold (LSB first: numpy's packbits(..., bitorder="little")).  Data are
 * 2-D C-contiguous float32, float16 or float64 tensors in host or device
 * memory; the uint8 output lives in the same kind of memory.  All compute
 * runs on the GPU (cuvs_b200/csrc/quantize.cu).  DESIGN.md "Quantizers"
 * states the thresholds.
 */
#pragma once
#include <cuvs/core/c_api.h>
#include <cuvs/core/export.h>
#include <dlpack/dlpack.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/** ZERO: every threshold is 0; MEAN: each column's mean; SAMPLING_MEDIAN: each column's median over a sample of rows. */
enum cuvsBinaryQuantizerThreshold { ZERO = 0, MEAN = 1, SAMPLING_MEDIAN = 2 };

struct cuvsBinaryQuantizerParams {
  enum cuvsBinaryQuantizerThreshold threshold; /* default MEAN */
  float sampling_ratio;                        /* share of rows SAMPLING_MEDIAN samples, in (0, 1]; default 0.1 */
};
typedef struct cuvsBinaryQuantizerParams* cuvsBinaryQuantizerParams_t;

CUVS_EXPORT cuvsError_t cuvsBinaryQuantizerParamsCreate(cuvsBinaryQuantizerParams_t* params);
CUVS_EXPORT cuvsError_t cuvsBinaryQuantizerParamsDestroy(cuvsBinaryQuantizerParams_t params);

typedef struct {
  uintptr_t addr;
  DLDataType dtype;
} cuvsBinaryQuantizer;
typedef cuvsBinaryQuantizer* cuvsBinaryQuantizer_t;

CUVS_EXPORT cuvsError_t cuvsBinaryQuantizerCreate(cuvsBinaryQuantizer_t* quantizer);
/** Frees the handle and its thresholds. */
CUVS_EXPORT cuvsError_t cuvsBinaryQuantizerDestroy(cuvsBinaryQuantizer_t quantizer);

CUVS_EXPORT cuvsError_t cuvsBinaryQuantizerTrain(cuvsResources_t res, cuvsBinaryQuantizerParams_t params, DLManagedTensor* dataset,
                                                 cuvsBinaryQuantizer_t quantizer);

/** Packs the signs of `dataset` (threshold ZERO) into `out`: uint8, at least n rows and ceil(dim / 8) columns.  Padding bits
 *  and bytes past ceil(dim / 8) are written as zero; rows past n are left untouched. */
CUVS_EXPORT cuvsError_t cuvsBinaryQuantizerTransform(cuvsResources_t res, DLManagedTensor* dataset, DLManagedTensor* out);

/** As cuvsBinaryQuantizerTransform, against a trained quantizer's thresholds.  `dataset` must have the type the quantizer
 *  was trained on and, for MEAN and SAMPLING_MEDIAN, as many columns as it has thresholds. */
CUVS_EXPORT cuvsError_t cuvsBinaryQuantizerTransformWithParams(cuvsResources_t res, cuvsBinaryQuantizer_t quantizer,
                                                               DLManagedTensor* dataset, DLManagedTensor* out);

#ifdef __cplusplus
}
#endif
