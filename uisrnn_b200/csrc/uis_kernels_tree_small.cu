#include "uis_launch.cuh"
#include "uis_beam_tree.cuh"
namespace uis {
// spill: the kernel whose tree-sized arrays live in p.tree_arena.
bool launch_tree_small(int H, int D, bool spill, const BeamParams& p, int ctas, unsigned smem, cudaStream_t st,
                       cudaError_t* err) {
  return with_shape(SmallShapes{}, H, D, [&](auto s) {
    using S = decltype(s);
    constexpr int block = Cfg<S::H, S::D, tree_cp<S::H>()>::BLOCK;
    auto kern = p.depth > 1 ? (spill ? uis_beam_tree_kernel<S::H, S::D, true, true>
                                     : uis_beam_tree_kernel<S::H, S::D, true, false>)
                            : (spill ? uis_beam_tree_kernel<S::H, S::D, false, true>
                                     : uis_beam_tree_kernel<S::H, S::D, false, false>);
    *err = launch_with_smem(kern, p, ctas, block, smem, st);
  });
}
}  // namespace uis
