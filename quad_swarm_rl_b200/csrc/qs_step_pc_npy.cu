// Step kernels of the control modes of qs_set_control on the numpy dynamics path (qs_set_numpy_dynamics): qs_step_pc.cu
// with the numpy path's floor model, as qs_step_kernel_pc_npy in namespace qs_pc_npy.
#define QS_NUMPY_DYNAMICS 1
#include "qs_step_pc.cu"
