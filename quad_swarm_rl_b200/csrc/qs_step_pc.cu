// Step kernels of the control modes of qs_set_control (QS_CONTROL_RAW_UNIT: raw_control_zero_middle=False;
// QS_CONTROL_POSITION: raw_control=False): qs_step.cuh's step kernel compiled once more with QS_CONTROL_MODES, which maps
// actions to motor commands by StepParams.control, and its select_step_kernel (qs_step_select.cuh), which instantiates
// only the single-warp shape with the grid-wide wait.  A translation unit of its own, with its symbols in namespace qs_pc,
// for the reason given in qs_step_npy.cu: the default kernels keep their machine code.  qs_step_pc_npy.cu includes this
// file with QS_NUMPY_DYNAMICS = 1 for the numpy dynamics path (namespace qs_pc_npy).
#define QS_CONTROL_MODES 1
#if QS_NUMPY_DYNAMICS
#define qs qs_pc_npy
#define qs_step_kernel qs_step_kernel_pc_npy
#else
#define qs qs_pc
#define qs_step_kernel qs_step_kernel_pc
#endif
#include "qs_step_select.cuh"
