// kernels_f64.cu -- the parity gate: the same kernels for Real = double, keeping the
// reference's f64 formulas verbatim.  Compiled with -fmad=false so that products and
// sums round like the reference's (rustc does not contract a*b+c).
#include "features.cuh"
#include "launch_impl.cuh"
namespace rptb {
RPTB_DEFINE_LAUNCHERS(f64, double)
cudaError_t launch_features_f64(const SceneView<double>& sv, const RenderArgs<double>& args, int features, double* acc, cudaStream_t stream) {
    return launch_features_impl<double>(sv, args, features, acc, stream);
}
}
