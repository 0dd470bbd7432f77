// GEMM kernel instantiations: f16 operands, A MN-major.
#include "gemm_kernel.cuh"

namespace ft {
template const void* gemm_kernel_ptr<FMT_F16, 1>(int, int, int, int);
}  // namespace ft
