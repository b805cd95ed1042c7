// Step kernels of the reference's numpy dynamics path (qs_set_numpy_dynamics; use_numba=False): qs_step.cuh's step kernel,
// compiled once more with the numpy path's floor model (QS_NUMPY_DYNAMICS, qs_device.cuh), in every shape of the default
// kernels.  A translation unit of its own, with its symbols in namespace qs_npy: compiled into quadswarm.cu's, the extra
// kernels change the register allocation of the default ones (their shared out-of-line device functions and the order in
// which the compiler meets them).
#define QS_NUMPY_DYNAMICS 1
#define qs qs_npy
#define qs_step_kernel qs_step_kernel_npy
#include "qs_step.cuh"

namespace qs {

#include "qs_step_select.cuh"

void* step_kernel_npy(int NP, bool split, bool scn, bool ho, bool dyn, bool nz) {
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
