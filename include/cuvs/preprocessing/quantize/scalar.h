/*
 * Scalar quantizer C boundary: float rows to int8 codes and back.
 * Same ABI as the reference's c/include/cuvs/preprocessing/quantize/scalar.h
 * (params struct, the plain host quantizer struct, Create/Destroy family,
 * Train, Transform, InverseTransform).
 *
 * Data are 2-D C-contiguous float32, float16 or float64 tensors (int8 for the
 * inverse's input) in host or device memory; an output lives in the same kind
 * of memory as its input.  All compute runs on the GPU
 * (cuvs_b200/csrc/quantize.cu); host data are streamed through device
 * buffers and the call returns once the host output is written.  DESIGN.md
 * "Quantizers" states the arithmetic.
 */
#pragma once
#include <cuvs/core/c_api.h>
#include <cuvs/core/export.h>
#include <dlpack/dlpack.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

struct cuvsScalarQuantizerParams {
  float quantile; /* share of the values kept between min_ and max_, in (0, 1]; default 0.99 */
};
typedef struct cuvsScalarQuantizerParams* cuvsScalarQuantizerParams_t;

CUVS_EXPORT cuvsError_t cuvsScalarQuantizerParamsCreate(cuvsScalarQuantizerParams_t* params);
CUVS_EXPORT cuvsError_t cuvsScalarQuantizerParamsDestroy(cuvsScalarQuantizerParams_t params);

/** The trained range: values of the training data's type, held exactly as doubles.  Create zero-fills it. */
typedef struct {
  double min_;
  double max_;
} cuvsScalarQuantizer;
typedef cuvsScalarQuantizer* cuvsScalarQuantizer_t;

CUVS_EXPORT cuvsError_t cuvsScalarQuantizerCreate(cuvsScalarQuantizer_t* quantizer);
CUVS_EXPORT cuvsError_t cuvsScalarQuantizerDestroy(cuvsScalarQuantizer_t quantizer);

/** Sets min_ / max_ to the lower / upper `quantile` bounds of a sample of `dataset`'s values.  Waits for the stream. */
CUVS_EXPORT cuvsError_t cuvsScalarQuantizerTrain(cuvsResources_t res, cuvsScalarQuantizerParams_t params, DLManagedTensor* dataset,
                                                 cuvsScalarQuantizer_t quantizer);

/** `out` (int8, the shape of `dataset`) receives the codes of `dataset`'s values. */
CUVS_EXPORT cuvsError_t cuvsScalarQuantizerTransform(cuvsResources_t res, cuvsScalarQuantizer_t quantizer, DLManagedTensor* dataset,
                                                     DLManagedTensor* out);

/** `out` (float32, float16 or float64, the shape of `dataset`) receives the values the int8 codes in `dataset` stand for. */
CUVS_EXPORT cuvsError_t cuvsScalarQuantizerInverseTransform(cuvsResources_t res, cuvsScalarQuantizer_t quantizer,
                                                            DLManagedTensor* dataset, DLManagedTensor* out);

#ifdef __cplusplus
}
#endif
