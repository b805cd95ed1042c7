// Which step-kernel instantiation a launch takes (host code; included by quadswarm.cu for qs_step_kernel, and by
// qs_step_npy.cu, where qs_step_kernel names the numpy dynamics path's kernels).
#pragma once

using KernelFn = void (*)(StepParams);

template <int NP, bool SPLIT, bool HO, bool DYN, bool NZ>
static KernelFn step_kernel_scn(bool scn) {
    return scn ? (KernelFn)qs_step_kernel<NP, SPLIT, true, HO, DYN, NZ> : (KernelFn)qs_step_kernel<NP, SPLIT, false, HO, DYN, NZ>;
}

// The step-kernel instantiation of a launch.  DYN and NZ exist only in the single-warp shape with the grid-wide wait, so
// `split` and `ho` do not apply to them.
template <int NP>
static KernelFn step_kernel(bool split, bool scn, bool ho, bool dyn, bool nz) {
    if (nz) return dyn ? step_kernel_scn<NP, false, false, true, true>(scn) : step_kernel_scn<NP, false, false, false, true>(scn);
    if (dyn) return step_kernel_scn<NP, false, false, true, false>(scn);
    if (split) return ho ? step_kernel_scn<NP, true, true, false, false>(scn) : step_kernel_scn<NP, true, false, false, false>(scn);
    return ho ? step_kernel_scn<NP, false, true, false, false>(scn) : step_kernel_scn<NP, false, false, false, false>(scn);
}
