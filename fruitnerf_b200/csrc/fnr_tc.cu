// Dispatch of impl = tcgen05 (the tensor-core implementation) on sm_90a.
//
// The field MLPs of render / export forward and of the field backward run on the Hopper tensor cores: fnr_simt.cu's
// kernels instantiated with WgmmaLinear / WgmmaBackward (fnr_wgmma.cuh: bf16 hi/lo split operands, wgmma, fp32
// accumulation; the backward's dx = W^T dy and per-tile dW = dY^T X as well), followed by the compositing kernel for
// render calls.  impl = auto takes them for both shipped families.  The name is the historical one: the fused Blackwell
// (tcgen05 / tensor memory) kernels this impl first selected are kept as a design record under design/blackwell/ and are
// not part of the library.
#include "fnr_common.cuh"
#include "fnr_kernels.h"

namespace fnr {

// auto takes the tensor-core kernels for both shipped families (4096x192 bench batch on an H100: render forward 1.4 ms
// against 3.7 ms on the simt kernels for fruit_nerf, 5.5 against 8.4 ms for fruit_nerf_big)
static bool shipped(Family fam) { return fam == kFamilySmall || fam == kFamilyBig; }
bool tc_supported(Family fam, const KField&, const KRays&) { return shipped(fam); }
bool tc_export_supported(Family fam, const KExport&) { return shipped(fam); }
bool tc_backward_supported(Family fam, const KField&, const KRays&, const KFieldBwd&) { return shipped(fam); }

int launch_tc_render_forward(Family fam, const KField& F, const KParams& P, const KRays& Rr, const KFieldOut& O, const KComposite& Cm,
                             cudaStream_t st) {
  const bool composite = Cm.rgb || Cm.accumulation || Cm.depth || Cm.depth_index || Cm.semantics || Cm.weights;
  if (composite && !(O.sample_density && O.sample_rgb && O.sample_semantics)) {
    set_error("tensor-core render: sample_density/sample_rgb/sample_semantics buffers are required when ray outputs are requested");
    return FNR_ERR_INVALID_ARGUMENT;
  }
  int rc = launch_wgmma_field_forward(fam, F, P, Rr, O, st);
  if (rc || !composite) return rc;
  return launch_simt_composite(Rr, Cm, st);
}

int launch_tc_export(Family fam, const KField& F, const KParams& P, const KExport& E, cudaStream_t st) {
  return launch_wgmma_export(fam, F, P, E, st);
}

int launch_tc_field_backward(Family fam, const KField& F, const KParams& P, const KParams& G, const KRays& Rr, const KFieldBwd& B,
                             cudaStream_t st) {
  return launch_wgmma_field_backward(fam, F, P, G, Rr, B, st);
}

}  // namespace fnr
