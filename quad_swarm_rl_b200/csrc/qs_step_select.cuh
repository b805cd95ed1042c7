// Which step-kernel instantiation a launch takes (host code).  Every translation unit with step kernels includes this file
// and so exports select_step_kernel in its own namespace, over its own qs_step_kernel: qs (quadswarm.cu), qs_npy
// (qs_step_npy.cu), and qs_pc and qs_pc_npy (qs_step_pc.cu, qs_step_pc_npy.cu).  plan_step (quadswarm.cu) picks the unit.
#pragma once
#include "qs_step.cuh"

namespace qs {

using KernelFn = void (*)(StepParams);

template <int NP, bool SPLIT, bool HO, bool DYN, bool NZ>
static KernelFn step_kernel_scn(bool scn) {
    return scn ? (KernelFn)qs_step_kernel<NP, SPLIT, true, HO, DYN, NZ> : (KernelFn)qs_step_kernel<NP, SPLIT, false, HO, DYN, NZ>;
}

// DYN, NZ and the control modes exist only in the single-warp shape with the grid-wide wait, so `split` and `ho` do not
// apply to them; the control-mode units (QS_CONTROL_MODES) do not instantiate the split and hand-over kernels at all and
// return the grid-wide-wait single-warp kernel whatever `split` and `ho` say.  The order in which the instantiations are
// named is the order in which the compiler meets them, which moves the register allocation of the kernels (DESIGN.md,
// "Numpy dynamics path"): keep it.
template <int NP>
static KernelFn step_kernel(bool split, bool scn, bool ho, bool dyn, bool nz) {
    if (nz) return dyn ? step_kernel_scn<NP, false, false, true, true>(scn) : step_kernel_scn<NP, false, false, false, true>(scn);
    if (dyn) return step_kernel_scn<NP, false, false, true, false>(scn);
    if constexpr (!QS_CONTROL_MODES) {
        if (split) return ho ? step_kernel_scn<NP, true, true, false, false>(scn) : step_kernel_scn<NP, true, false, false, false>(scn);
        if (ho) return step_kernel_scn<NP, false, true, false, false>(scn);
    }
    return step_kernel_scn<NP, false, false, false, false>(scn);
}

// The step kernel of a launch, as a void* because StepParams is a type of the unit's own namespace.
void* select_step_kernel(int NP, bool split, bool scn, bool ho, bool dyn, bool nz) {
    switch (NP) {
        case 1: return (void*)step_kernel<1>(split, scn, ho, dyn, nz);
        case 2: return (void*)step_kernel<2>(split, scn, ho, dyn, nz);
        case 4: return (void*)step_kernel<4>(split, scn, ho, dyn, nz);
        case 8: return (void*)step_kernel<8>(split, scn, ho, dyn, nz);
        case 16: return (void*)step_kernel<16>(split, scn, ho, dyn, nz);
        case 32: return (void*)step_kernel<32>(split, scn, ho, dyn, nz);
    }
    return nullptr;       // qs_create takes N <= 32 only, rounded up to these group sizes
}

}  // namespace qs
