// Host-visible interface of the fused worker-step kernel (fused_step_sm90.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "protocol.h"

namespace dm {

struct FusedMaps {
  CUtensorMap w[kFusedCluster];  // hidden weight [H][I] on the shard that owns CTA r's slice (box 32 x 128)
  CUtensorMap xk;                // x (box 32 features x 32 rows, SWIZZLE_128B): forward B operand and dW A operand
  CUtensorMap push[kFusedCluster];  // where CTA r's dW tile goes: [slot][H][I] view of this worker's mailbox for the
                                    // hidden weight on the owning shard (mailbox mode) or of the master copy (atomic
                                    // mode, 1 slot); box 32 x 128 x 1, SWIZZLE_128B — destination of the TMA store
};

// Whether a step runs the general-head instantiations: under an activation other than the ReLU, a loss after LOSS_XENT
// or a label smoothing (FusedParams::act, loss_kind, label_smoothing).
inline bool fused_general_head(int act, int loss_kind, float label_smoothing) {
  return act > ACT_RELU || loss_kind > LOSS_XENT || label_smoothing != 0.f;
}

// Batch B <= 32 runs the one-tile instantiation of the kernel, 32 < B <= 256 the multi-tile one; the functions that
// take B answer for the instantiation that batch runs, with (clip) or without gradient clipping, with (l2) or without
// L2 regularization, with (general) or without the general head.
size_t fused_smem_bytes(int B);
cudaError_t launch_fused_step(const FusedMaps& maps, const FusedParams& p, int lanes, cudaStream_t stream);
// how many clusters of that instantiation can be co-resident on the device (upper bound for `lanes`)
cudaError_t fused_max_lanes(int B, bool clip, bool l2, bool general, int* out);

}  // namespace dm
