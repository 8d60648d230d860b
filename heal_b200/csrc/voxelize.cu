// GPU voxelizer: bit-exact, order-preserving restatement of the spconv CPU voxel generator that
// the reference calls from SpVoxelPreprocessor.preprocess
// (reference: opencood/data_utils/pre_processor/sp_voxel_preprocessor.py:62-85; algorithm = spconv
// `points_to_voxel_3d_np`, see oracle/voxelizer.c and DESIGN.md).
//
// The CPU algorithm is sequential and order dependent:
//   voxel id        = order of first appearance of the cell in the point array,
//   slot in a voxel = order of appearance of the point among the points of that cell (first T kept),
//   cells whose first appearance comes after `max_voxels` cells already exist are dropped.
// Parallel formulation (all agents of a scene in one batch of launches):
//   1. cell key per point + hash insert with atomicMin(first point index)          [k_cells_insert]
//   2. flag(point is the first of its cell) -> exclusive scan -> appearance rank     [scan]
//   3. per-agent clamp to max_voxels, output base per agent, voxel id per cell       [k_agent_bases, k_assign]
//   4. per-voxel point count -> scan -> CSR fill (unordered)                         [k_count, scan, k_fill]
//   5. one warp per voxel selects the T smallest point indices in ascending order    [k_select]
// Agent a owns rows [offs[a], offs[a+1]); rows outside [offs[0], offs[A]) are ignored.  Voxel rows at or past `capacity` are
// dropped (not written, their points not counted), while num_voxels_out keeps the true counts.
// Every step is deterministic in its OUTPUT (atomics only build unordered sets that are ordered
// afterwards), so indices/counts/features are bit-exact with the CPU generator.
#include "common.cuh"
#include "../../include/heal_b200.h"

namespace {

constexpr uint32_t KEY_EMPTY = 0xFFFFFFFFu;
constexpr int SCAN_BLOCK = 1024;

struct VoxCfg {
    float minx, miny, minz;
    float vsx, vsy, vsz;
    int gx, gy, gz;
    int T, maxV, A, P, cap;
    uint32_t cells;     // gx*gy*gz
    uint32_t tmask;     // hash table size - 1
    int tshift;         // 32 - log2(table size)
};

__device__ __forceinline__ int find_agent(const int* __restrict__ offs, int A, int i) {
    int a = 0;
    while (a + 1 < A && i >= offs[a + 1]) ++a;
    return a;
}

__global__ void k_cells_insert(const float4* __restrict__ pts, const int* __restrict__ offs, VoxCfg c,
                               uint32_t* __restrict__ keys, int* __restrict__ firsts, int* __restrict__ pt_slot) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c.P) return;
    // `P` may be the CAPACITY of a static (CUDA-graph) input buffer: the live point count is offs[A] on the device.
    // Rows before offs[0] belong to no agent.
    if (i < offs[0] || i >= offs[c.A]) { pt_slot[i] = -1; return; }
    float4 p = __ldg(pts + i);
    // IEEE fp32 subtract + divide + floor, exactly as the CPU generator (no reciprocal multiply).
    float fx = floorf(__fdiv_rn(__fsub_rn(p.x, c.minx), c.vsx));
    float fy = floorf(__fdiv_rn(__fsub_rn(p.y, c.miny), c.vsy));
    float fz = floorf(__fdiv_rn(__fsub_rn(p.z, c.minz), c.vsz));
    bool ok = (fx >= 0.f) && (fx < (float)c.gx) && (fy >= 0.f) && (fy < (float)c.gy) && (fz >= 0.f) && (fz < (float)c.gz);
    if (!ok) { pt_slot[i] = -1; return; }
    int a = find_agent(offs, c.A, i);
    uint32_t cell = ((uint32_t)fz * (uint32_t)c.gy + (uint32_t)fy) * (uint32_t)c.gx + (uint32_t)fx;
    uint32_t key = (uint32_t)a * c.cells + cell;
    uint32_t slot = (key * 2654435761u) >> c.tshift;
    while (true) {
        uint32_t prev = atomicCAS(&keys[slot], KEY_EMPTY, key);
        if (prev == KEY_EMPTY || prev == key) break;
        slot = (slot + 1) & c.tmask;
    }
    atomicMin(&firsts[slot], i);
    pt_slot[i] = (int)slot;
}

// ---- exclusive scan (two-level; n <= 1024*1024) -------------------------------------------------
// MODE 0: value = in[i];  MODE 1: value = (pt_slot[i] >= 0 && firsts[pt_slot[i]] == i)
template <int MODE>
__global__ void k_scan_local(const int* __restrict__ in, const int* __restrict__ firsts, int n,
                             int* __restrict__ local_excl, int* __restrict__ block_sums) {
    __shared__ int warp_tot[32];
    int i = blockIdx.x * SCAN_BLOCK + threadIdx.x;
    int v = 0;
    if (i < n) {
        if (MODE == 0) v = in[i];
        else { int s = in[i]; v = (s >= 0 && firsts[s] == i) ? 1 : 0; }
    }
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    if (w == 0) {
        int t = warp_tot[lane];
        int ti = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += u; }
        warp_tot[lane] = ti - t;  // exclusive warp offsets
        if (lane == 31) block_sums[blockIdx.x] = ti;
    }
    __syncthreads();
    if (i < n) local_excl[i] = inc - v + warp_tot[w];
}

__global__ void k_scan_blocks(int* __restrict__ block_sums, int nblocks) {
    // single block of 1024 threads; in-place exclusive scan of block_sums, total at [nblocks]
    __shared__ int warp_tot[32];
    int t = threadIdx.x;
    int v = (t < nblocks) ? block_sums[t] : 0;
    int lane = t & 31, w = t >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += u; }
    if (lane == 31) warp_tot[w] = inc;
    __syncthreads();
    if (w == 0) {
        int x = warp_tot[lane];
        int xi = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, xi, o); if (lane >= o) xi += u; }
        warp_tot[lane] = xi - x;
    }
    __syncthreads();
    int excl = inc - v + warp_tot[w];
    if (t < nblocks) block_sums[t] = excl;
    if (t == nblocks - 1) block_sums[nblocks] = excl + v;
}

__device__ __forceinline__ int scan_at(const int* local_excl, const int* block_off, int i, int n, int nblocks) {
    return (i >= n) ? block_off[nblocks] : local_excl[i] + block_off[i / SCAN_BLOCK];
}

// per agent: rank of its first voxel, number of kept voxels, output base. meta layout:
//   meta[0..A]      first_rank (rank at offs[a]; meta[A] = total cells)
//   meta[A+1..2A+1] out_base   (meta[2A+1] = M_total)
// num_voxels_out[0] = M_total, [1+a] = kept voxels of agent a
__global__ void k_agent_bases(const int* __restrict__ offs, const int* __restrict__ local_excl,
                              const int* __restrict__ block_off, VoxCfg c, int nblocks,
                              int* __restrict__ meta, int* __restrict__ num_voxels_out) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    for (int a = 0; a <= c.A; ++a) meta[a] = scan_at(local_excl, block_off, (a == c.A) ? c.P : offs[a], c.P, nblocks);
    int base = 0;
    for (int a = 0; a < c.A; ++a) {
        int nv = min(meta[a + 1] - meta[a], c.maxV);
        meta[c.A + 1 + a] = base;
        num_voxels_out[1 + a] = nv;
        base += nv;
    }
    meta[2 * c.A + 1] = base;
    num_voxels_out[0] = base;
}

__global__ void k_assign(const int* __restrict__ offs, const int* __restrict__ pt_slot, const int* __restrict__ firsts,
                         const uint32_t* __restrict__ keys, const int* __restrict__ local_excl,
                         const int* __restrict__ block_off, const int* __restrict__ meta, VoxCfg c,
                         int* __restrict__ slot_vid, int* __restrict__ coords) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c.P) return;
    int s = pt_slot[i];
    if (s < 0 || firsts[s] != i) return;
    int a = find_agent(offs, c.A, i);
    int rank = local_excl[i] + block_off[i / SCAN_BLOCK];
    int local = rank - meta[a];
    int vid = (local < c.maxV) ? (meta[c.A + 1 + a] + local) : -1;
    if (vid >= c.cap) vid = -1;   // rows past the output capacity are dropped; num_voxels_out still counts them
    slot_vid[s] = vid;
    if (vid >= 0) {
        uint32_t cell = keys[s] - (uint32_t)a * c.cells;
        int x = (int)(cell % (uint32_t)c.gx);
        int y = (int)((cell / (uint32_t)c.gx) % (uint32_t)c.gy);
        int z = (int)(cell / ((uint32_t)c.gx * (uint32_t)c.gy));
        reinterpret_cast<int4*>(coords)[vid] = make_int4(a, z, y, x);  // [batch, z, y, x]
    }
}

__global__ void k_count(const int* __restrict__ pt_slot, const int* __restrict__ slot_vid, int P,
                        int* __restrict__ pt_vid, int* __restrict__ cnt) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    int s = pt_slot[i];
    int vid = (s >= 0) ? slot_vid[s] : -1;
    pt_vid[i] = vid;
    if (vid >= 0) atomicAdd(&cnt[vid], 1);
}

__global__ void k_fill(const int* __restrict__ pt_vid, int P, const int* __restrict__ seg_local,
                       const int* __restrict__ seg_blockoff, int* __restrict__ cursor, int* __restrict__ seg) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    int vid = pt_vid[i];
    if (vid < 0) return;
    int pos = seg_local[vid] + seg_blockoff[vid / SCAN_BLOCK] + atomicAdd(&cursor[vid], 1);
    seg[pos] = i;
}

// One warp per voxel: order the voxel's point indices ascending, keep the first T, write the
// zero-padded (T,4) feature block and the point count.
__global__ void k_select(const float4* __restrict__ pts, const int* __restrict__ seg, const int* __restrict__ cnt,
                         const int* __restrict__ seg_local, const int* __restrict__ seg_blockoff,
                         const int* __restrict__ num_voxels, int T, int cap,
                         float4* __restrict__ voxels, int* __restrict__ num_points) {
    // persistent warps: the launch is sized for the machine, not for the row CAPACITY (the live voxel count is on the device
    // and typically 4-5x below the capacity: a capacity-sized grid spent most of its blocks on an early exit)
    const int lane = threadIdx.x & 31;
    const int nv = min(num_voxels[0], cap);
    const int wstride = (gridDim.x * blockDim.x) >> 5;
    for (int v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < nv; v += wstride) {
    int n = cnt[v];
    int base = seg_local[v] + seg_blockoff[v / SCAN_BLOCK];
    int m = min(n, T);
    float4* out = voxels + (size_t)v * T;
    const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
    if (n <= 32) {
        int idx = (lane < n) ? seg[base + lane] : 0x7fffffff;
        int rank = 0;
        for (int j = 0; j < n; ++j) { int o = __shfl_sync(0xffffffffu, idx, j); rank += (o < idx) ? 1 : 0; }
        if (lane < n && rank < T) out[rank] = __ldg(pts + idx);
        for (int s = m + lane; s < T; s += 32) out[s] = zero;
    } else {
        int prev = -1;
        for (int r0 = 0; r0 < T; r0 += 32) {
            int mine = -1;  // point index selected for slot r0+lane
            int rounds = min(32, T - r0);
            for (int r = 0; r < rounds; ++r) {
                int best = 0x7fffffff;
                if (r0 + r < m) {
                    for (int j = lane; j < n; j += 32) { int o = seg[base + j]; if (o > prev && o < best) best = o; }
                    best = warp_min_i(best);
                    prev = best;
                }
                if (lane == r) mine = (r0 + r < m) ? best : -1;
            }
            int s = r0 + lane;
            if (s < T) out[s] = (mine >= 0) ? __ldg(pts + mine) : zero;
        }
    }
    if (lane == 0) num_points[v] = m;
    }
}

__global__ void k_mean_vfe(const float4* __restrict__ voxels, const int* __restrict__ num_points, int M, int T,
                           float4* __restrict__ out) {
    int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= M) return;
    float sx = 0.f, sy = 0.f, sz = 0.f, sw = 0.f;
    for (int t = 0; t < T; ++t) {  // sequential sum over all T slots like torch.sum(dim=1) on a (T,4) row
        float4 p = __ldg(voxels + (size_t)v * T + t);
        sx += p.x; sy += p.y; sz += p.z; sw += p.w;
    }
    float nrm = fmaxf((float)num_points[v], 1.0f);
    out[v] = make_float4(__fdiv_rn(sx, nrm), __fdiv_rn(sy, nrm), __fdiv_rn(sz, nrm), __fdiv_rn(sw, nrm));
}

int table_log2(int P) {
    int lg = 10;
    while ((1 << lg) < 2 * P) ++lg;
    return lg;
}

}  // namespace

extern "C" size_t heal_voxelize_workspace(int num_points_total, int capacity, int num_agents) {
    size_t P = (size_t)(num_points_total > 0 ? num_points_total : 1), cap = (size_t)(capacity > 0 ? capacity : 1);
    size_t tsize = (size_t)1 << table_log2((int)P);
    size_t nb_p = (P + SCAN_BLOCK - 1) / SCAN_BLOCK + 2, nb_c = (cap + SCAN_BLOCK - 1) / SCAN_BLOCK + 2;
    size_t bytes = 0;
    bytes += heal_align_up(tsize * 4, 256) * 3;        // keys, firsts, slot_vid
    bytes += heal_align_up(P * 4, 256) * 4;            // pt_slot, pt_vid, local_excl, seg
    bytes += heal_align_up(cap * 4, 256) * 3;          // cnt, cursor, seg_local
    bytes += heal_align_up(nb_p * 4, 256) + heal_align_up(nb_c * 4, 256);
    bytes += heal_align_up((2 * (size_t)num_agents + 2) * 4, 256);
    return bytes + 4096;
}

extern "C" int heal_voxelize(const float* points, const int* agent_offsets, int num_agents, int num_points_total,
                             const float* range_min3, const float* voxel_size3, const int* grid3,
                             int max_points_per_voxel, int max_voxels, int capacity,
                             float* voxels_out, int* coords_out, int* num_points_out, int* num_voxels_out,
                             void* workspace, size_t workspace_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!points || !agent_offsets || !voxels_out || !coords_out || !num_points_out || !num_voxels_out) return HEAL_ERR_ARG;
    if (num_agents < 1 || num_agents > 64 || max_points_per_voxel < 1 || max_voxels < 1 || capacity < 1) return HEAL_ERR_ARG;
    if (num_points_total < 0 || num_points_total > SCAN_BLOCK * SCAN_BLOCK || capacity > SCAN_BLOCK * SCAN_BLOCK) return HEAL_ERR_ARG;
    unsigned long long cells = (unsigned long long)grid3[0] * grid3[1] * grid3[2];
    if (grid3[0] < 1 || grid3[1] < 1 || grid3[2] < 1 || cells * (unsigned long long)num_agents >= 0xFFFFFFFFull) return HEAL_ERR_ARG;
    if (workspace_bytes < heal_voxelize_workspace(num_points_total, capacity, num_agents)) return HEAL_ERR_WORKSPACE;
    const int P = num_points_total, A = num_agents;
    if (P == 0) {
        cudaMemsetAsync(num_voxels_out, 0, sizeof(int) * (1 + A), st);
        return heal_check_launch();
    }
    VoxCfg c;
    c.minx = range_min3[0]; c.miny = range_min3[1]; c.minz = range_min3[2];
    c.vsx = voxel_size3[0]; c.vsy = voxel_size3[1]; c.vsz = voxel_size3[2];
    c.gx = grid3[0]; c.gy = grid3[1]; c.gz = grid3[2];
    c.T = max_points_per_voxel; c.maxV = max_voxels; c.A = A; c.P = P; c.cap = capacity;
    c.cells = (uint32_t)cells;
    int lg = table_log2(P);
    size_t tsize = (size_t)1 << lg;
    c.tmask = (uint32_t)(tsize - 1);
    c.tshift = 32 - lg;

    HealArena ar(workspace, workspace_bytes);
    uint32_t* keys = ar.take<uint32_t>(tsize);
    int* firsts = ar.take<int>(tsize);
    int* slot_vid = ar.take<int>(tsize);
    int* pt_slot = ar.take<int>(P);
    int* pt_vid = ar.take<int>(P);
    int* local_excl = ar.take<int>(P);
    int* seg = ar.take<int>(P);
    int* cnt = ar.take<int>(capacity);
    int* cursor = ar.take<int>(capacity);
    int* seg_local = ar.take<int>(capacity);
    int nb_p = (P + SCAN_BLOCK - 1) / SCAN_BLOCK, nb_c = (capacity + SCAN_BLOCK - 1) / SCAN_BLOCK;
    int* block_off = ar.take<int>(nb_p + 2);
    int* seg_blockoff = ar.take<int>(nb_c + 2);
    int* meta = ar.take<int>(2 * A + 2);
    if (!ar.ok()) return HEAL_ERR_WORKSPACE;

    cudaMemsetAsync(keys, 0xFF, tsize * 4, st);
    cudaMemsetAsync(firsts, 0x7F, tsize * 4, st);
    cudaMemsetAsync(cnt, 0, (size_t)capacity * 4, st);
    cudaMemsetAsync(cursor, 0, (size_t)capacity * 4, st);

    const int TB = 256;
    int gp = (P + TB - 1) / TB;
    k_cells_insert<<<gp, TB, 0, st>>>((const float4*)points, agent_offsets, c, keys, firsts, pt_slot);
    k_scan_local<1><<<nb_p, SCAN_BLOCK, 0, st>>>(pt_slot, firsts, P, local_excl, block_off);
    k_scan_blocks<<<1, SCAN_BLOCK, 0, st>>>(block_off, nb_p);
    k_agent_bases<<<1, 32, 0, st>>>(agent_offsets, local_excl, block_off, c, nb_p, meta, num_voxels_out);
    k_assign<<<gp, TB, 0, st>>>(agent_offsets, pt_slot, firsts, keys, local_excl, block_off, meta, c, slot_vid, coords_out);
    k_count<<<gp, TB, 0, st>>>(pt_slot, slot_vid, P, pt_vid, cnt);
    k_scan_local<0><<<nb_c, SCAN_BLOCK, 0, st>>>(cnt, nullptr, capacity, seg_local, seg_blockoff);
    k_scan_blocks<<<1, SCAN_BLOCK, 0, st>>>(seg_blockoff, nb_c);
    k_fill<<<gp, TB, 0, st>>>(pt_vid, P, seg_local, seg_blockoff, cursor, seg);
    int gv = (int)(((size_t)capacity * 32 + TB - 1) / TB);
    if (gv > HEAL_NUM_SMS * 8) gv = HEAL_NUM_SMS * 8;           // 8 resident blocks of 8 warps per SM, warp-stride loop over the voxels
    k_select<<<gv, TB, 0, st>>>((const float4*)points, seg, cnt, seg_local, seg_blockoff, num_voxels_out,
                                c.T, capacity, (float4*)voxels_out, num_points_out);
    return heal_check_launch(10);
}

extern "C" int heal_mean_vfe(const float* voxels, const int* num_points, int num_voxels, int max_points_per_voxel,
                             float* mean_out, void* stream_) {
    if (num_voxels <= 0) return HEAL_OK;
    if (!voxels || !num_points || !mean_out || max_points_per_voxel < 1) return HEAL_ERR_ARG;
    k_mean_vfe<<<(num_voxels + 127) / 128, 128, 0, (cudaStream_t)stream_>>>(
        (const float4*)voxels, num_points, num_voxels, max_points_per_voxel, (float4*)mean_out);
    return heal_check_launch();
}
