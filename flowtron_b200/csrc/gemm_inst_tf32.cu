// GEMM kernel instantiations: tf32 operands, A K-major.
#include "gemm_kernel.cuh"

namespace ft {
template const void* gemm_kernel_ptr<FMT_TF32, 0>(int, int, int, int);
}  // namespace ft
