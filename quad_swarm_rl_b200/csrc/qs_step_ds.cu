// The step kernels of handles with the device-side dynamics sampler (qs_set_dynamics_sampler): the DYN instantiations
// compiled with the sampler's reset path (QS_DYN_SAMPLER), in units of their own, so that the DYN kernels of every other
// handle keep their code.  This unit: njit dynamics path, RawControl; qs_step_ds_npy.cu, qs_step_ds_pc.cu and
// qs_step_ds_pc_npy.cu define QS_NUMPY_DYNAMICS / QS_CONTROL_MODES and include it.
#define QS_DYN_SAMPLER 1
#if defined(QS_CONTROL_MODES) && QS_CONTROL_MODES
#if defined(QS_NUMPY_DYNAMICS) && QS_NUMPY_DYNAMICS
#define qs qs_ds_pc_npy
#define qs_step_kernel qs_step_kernel_ds_pc_npy
#else
#define qs qs_ds_pc
#define qs_step_kernel qs_step_kernel_ds_pc
#endif
#elif defined(QS_NUMPY_DYNAMICS) && QS_NUMPY_DYNAMICS
#define qs qs_ds_npy
#define qs_step_kernel qs_step_kernel_ds_npy
#else
#define qs qs_ds
#define qs_step_kernel qs_step_kernel_ds
#endif
#include "qs_step_select.cuh"
