// The dynamics sampler's step kernels with the control modes, on the numpy dynamics path (see qs_step_ds.cu).
#define QS_CONTROL_MODES 1
#define QS_NUMPY_DYNAMICS 1
#include "qs_step_ds.cu"
