// The dynamics sampler's step kernels on the numpy dynamics path (see qs_step_ds.cu).
#define QS_NUMPY_DYNAMICS 1
#include "qs_step_ds.cu"
