// immesh_b200 -- programmatic dependent launch (Hopper): the device side of IM_LAUNCH_PDL (common_host.hpp).
// A kernel launched with IM_LAUNCH_PDL may be scheduled while its predecessor on the stream is still running.  pdl_wait() blocks
// until that predecessor has completed and its stores are visible, so results are those of an ordinary launch as long as
//   - a kernel launched with IM_LAUNCH_PDL calls pdl_wait() before its first global memory access, on every path (a kernel that
//     returns without waiting would let its own successor start before the predecessor has finished), and
//   - pdl_trigger() comes after the block's last global store; it only lets the successor's blocks be scheduled early.
// Both are no-ops for a kernel launched without the attribute, and compile to nothing outside device code.
#pragma once

namespace immesh {
__device__ __forceinline__ void pdl_wait() {
#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ >= 900
    asm volatile("griddepcontrol.wait;" ::: "memory");
#endif
}
__device__ __forceinline__ void pdl_trigger() {
#if defined(__CUDA_ARCH__) && __CUDA_ARCH__ >= 900
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
#endif
}
}  // namespace immesh
