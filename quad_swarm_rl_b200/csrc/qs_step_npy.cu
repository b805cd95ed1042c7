// Step kernels of the reference's numpy dynamics path (qs_set_numpy_dynamics; use_numba=False): qs_step.cuh's step kernel,
// compiled once more with the numpy path's floor model (QS_NUMPY_DYNAMICS, qs_device.cuh), in every shape of the default
// kernels, and their select_step_kernel (qs_step_select.cuh).  A translation unit of its own, with its symbols in namespace
// qs_npy: compiled into quadswarm.cu's, the extra kernels change the register allocation of the default ones (their shared
// out-of-line device functions and the order in which the compiler meets them).
#define QS_NUMPY_DYNAMICS 1
#define qs qs_npy
#define qs_step_kernel qs_step_kernel_npy
#include "qs_step_select.cuh"
