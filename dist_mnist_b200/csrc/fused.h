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

cudaError_t prepare_fused_kernel();
size_t fused_smem_bytes();
cudaError_t launch_fused_step(const FusedMaps& maps, const FusedParams& p, int lanes, cudaStream_t stream);
cudaError_t fused_max_lanes(int* out);

}  // namespace dm
