// Step kernels of the control modes of qs_set_control (QS_CONTROL_RAW_UNIT: raw_control_zero_middle=False;
// QS_CONTROL_POSITION: raw_control=False): qs_step.cuh's step kernel compiled once more with QS_CONTROL_MODES, which maps
// actions to motor commands by StepParams.control.  Only the single-warp shape with the grid-wide wait, with and without
// the device scenarios, per-drone constants (DYN) and the custom sensor-noise model (NZ).  A translation unit of its own,
// with its symbols in namespace qs_pc, for the reason given in qs_step_npy.cu: the default kernels keep their machine
// code.  qs_step_pc_npy.cu includes this file with QS_NUMPY_DYNAMICS = 1 for the numpy dynamics path (namespace qs_pc_npy).
#define QS_CONTROL_MODES 1
#if QS_NUMPY_DYNAMICS
#define qs qs_pc_npy
#define qs_step_kernel qs_step_kernel_pc_npy
#else
#define qs qs_pc
#define qs_step_kernel qs_step_kernel_pc
#endif
#include "qs_step.cuh"

namespace qs {

#include "qs_step_select.cuh"

template <int NP>
static KernelFn step_kernel_control(bool scn, bool dyn, bool nz) {
    if (nz) return dyn ? step_kernel_scn<NP, false, false, true, true>(scn) : step_kernel_scn<NP, false, false, false, true>(scn);
    return dyn ? step_kernel_scn<NP, false, false, true, false>(scn) : step_kernel_scn<NP, false, false, false, false>(scn);
}

void* step_kernel_pc(int NP, bool scn, bool dyn, bool nz) {
    switch (NP) {
        case 1: return (void*)step_kernel_control<1>(scn, dyn, nz);
        case 2: return (void*)step_kernel_control<2>(scn, dyn, nz);
        case 4: return (void*)step_kernel_control<4>(scn, dyn, nz);
        case 8: return (void*)step_kernel_control<8>(scn, dyn, nz);
        case 16: return (void*)step_kernel_control<16>(scn, dyn, nz);
        case 32: return (void*)step_kernel_control<32>(scn, dyn, nz);
    }
    return nullptr;       // qs_create takes N <= 32 only, rounded up to these group sizes
}

}  // namespace qs
