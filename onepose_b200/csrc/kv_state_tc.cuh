// wgmma linear-attention state kernel -- declarations.  See kv_state_tc.cu.
#pragma once
#include "common.cuh"

namespace opb {
// Row groups of the state kernel: every segment is cut into groups of `slabs` 256-row slabs; frame b owns groups
// [b*(gq+gd), +gq) (query side) and the next gd (3D side).  One partial state per group.
struct KvGroups {
  int gq, gd, slabs;
};
KvGroups kv_groups_for(const Layout& L, int num_sms);
// kvh = fp16 [rows, 512] = 64 * [elu1(K) | V] with pad rows zero (written by the k,v GEMM, EPI_QKV).
// partial: [B*(gq+gd)][4 heads][64*64 + 64] per-group sums (KV then Ksum), reduced per segment by kv_state_reduce.
// A tensor map the driver rejects is reported as cudaErrorInvalidValue.
cudaError_t launch_kv_state_h(const __half* kvh, const Layout& L, const KvGroups& G, float* partial, cudaStream_t stream);
}  // namespace opb
