// The dynamics sampler's step kernels with the control modes of qs_set_control (see qs_step_ds.cu).
#define QS_CONTROL_MODES 1
#include "qs_step_ds.cu"
