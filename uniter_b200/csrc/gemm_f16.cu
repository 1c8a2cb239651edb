// fp16 instantiations of the wgmma GEMM core (split from bf16 for build parallelism).
#include "gemm_impl.cuh"
namespace ub {
int gemm_dispatch_f16(int bn, int cluster, int a_major, int b_major, const GemmParams& p,
                      const CUtensorMap& tmA, const CUtensorMap& tmB, int grid, cudaStream_t stream) {
  return gemm_dispatch<false>(bn, cluster, a_major, b_major, p, tmA, tmB, grid, stream);
}
int gemm_group_dispatch_f16(const void* tm, const GroupedParams& g, int grid, cudaStream_t stream) {
  return gemm_group_dispatch<false>(*reinterpret_cast<const TmPack*>(tm), g, grid, stream);
}
}  // namespace ub
