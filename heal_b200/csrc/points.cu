// On-GPU input path (SURVEY.md 8f-4, first half): the point-cloud filters the reference applies on the host before voxelisation
// (opencood/data_utils/datasets/intermediate_heter_fusion_dataset.py:141-173 -> opencood/utils/pcd_utils.py):
//   shuffle_points          :91-95   points[np.random.permutation(n)]           -> `perm` (host-drawn indices, optional)
//   mask_ego_points         :70-88   drop -1.95 <= x <= 2.95 and -1.1 <= y <= 1.1
//   mask_points_by_range    :41-67   keep  min < p < max on x, y, z (strict)
// as ONE order-preserving compaction per agent: flags -> exclusive scan (CUB) -> scatter, new per-agent offsets on the device.
// Output order = the reference's (a stable filter of the permuted cloud), so the voxeliser downstream stays bit-exact.
#include <cub/cub.cuh>

#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

struct MaskP {
    const float4* pts; const int* perm; const int* offs; int A, P;
    float lo[3], hi[3]; int remove_ego;
};

__device__ __forceinline__ float4 src_point(const MaskP& p, int i) { return __ldg(p.pts + (p.perm ? p.perm[i] : i)); }

__global__ void k_mask_flags(MaskP p, int* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.P) return;
    int keep = 0;
    if (i >= p.offs[0] && i < p.offs[p.A]) {         // rows before offs[0] belong to no agent: the output offsets start at 0
        const float4 q = src_point(p, i);
        keep = (q.x > p.lo[0]) && (q.x < p.hi[0]) && (q.y > p.lo[1]) && (q.y < p.hi[1]) && (q.z > p.lo[2]) && (q.z < p.hi[2]);
        if (p.remove_ego && (q.x >= -1.95f) && (q.x <= 2.95f) && (q.y >= -1.1f) && (q.y <= 1.1f)) keep = 0;
    }
    flags[i] = keep;
}

__global__ void k_mask_scatter(MaskP p, const int* __restrict__ flags, const int* __restrict__ pos, float4* __restrict__ out,
                               int* __restrict__ offs_out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= p.A) {                      // new agent offsets: kept points before the agent's first point
        const int s = p.offs[i];
        offs_out[i] = (s < p.P) ? pos[s] : (p.P > 0 ? pos[p.P - 1] + flags[p.P - 1] : 0);
    }
    if (i >= p.P) return;
    if (flags[i]) out[pos[i]] = src_point(p, i);
}

}  // namespace

extern "C" size_t heal_mask_points_workspace(int num_points) {
    if (num_points < 1) num_points = 1;
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, (const int*)nullptr, (int*)nullptr, num_points);
    return heal_align_up((size_t)num_points * 4, 256) * 2 + heal_align_up(tb, 256) + 512;
}

extern "C" int heal_mask_points(const float* points, const int* perm, const int* agent_offsets, int num_agents, int num_points,
                                const float* range6_host, int remove_ego, float* points_out, int* agent_offsets_out,
                                void* workspace, size_t workspace_bytes, void* stream_) {
    if (!points || !agent_offsets || !range6_host || !points_out || !agent_offsets_out || !workspace) return HEAL_ERR_ARG;
    if (num_agents < 1 || num_agents > 64 || num_points < 0) return HEAL_ERR_ARG;
    if (workspace_bytes < heal_mask_points_workspace(num_points)) return HEAL_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream_;
    if (num_points == 0) { cudaMemsetAsync(agent_offsets_out, 0, sizeof(int) * (num_agents + 1), st); return heal_check_launch(0); }
    HealArena ar(workspace, workspace_bytes);
    int* flags = ar.take<int>(num_points);
    int* pos = ar.take<int>(num_points);
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, (const int*)nullptr, (int*)nullptr, num_points);
    char* tmp = ar.take<char>(tb);
    if (!ar.ok()) return HEAL_ERR_WORKSPACE;
    MaskP p;
    p.pts = (const float4*)points; p.perm = perm; p.offs = agent_offsets; p.A = num_agents; p.P = num_points;
    for (int j = 0; j < 3; ++j) { p.lo[j] = range6_host[j]; p.hi[j] = range6_host[3 + j]; }
    p.remove_ego = remove_ego;
    const unsigned g = (unsigned)((num_points + 255) / 256);
    k_mask_flags<<<g, 256, 0, st>>>(p, flags);
    if (cub::DeviceScan::ExclusiveSum(tmp, tb, flags, pos, num_points, st) != cudaSuccess) return HEAL_ERR_LAUNCH;
    k_mask_scatter<<<g, 256, 0, st>>>(p, flags, pos, (float4*)points_out, agent_offsets_out);
    return heal_check_launch(3);
}
