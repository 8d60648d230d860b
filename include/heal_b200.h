/* heal_b200 — C ABI of the H100-native (sm_90a) per-frame perception hot path of HEAL / OpenCOOD.
 *
 * The reference (yifanlu0227/HEAL) is pure Python/PyTorch on this path and has NO foreign-function
 * interface of its own; each entry point below therefore cites the reference *Python* call site it
 * replaces (path:line relative to the reference root). INTEGRATION.md shows the ctypes binding a
 * maintainer adds on the reference side.
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer is a DEVICE pointer unless the name ends in _host
 *    or the comment says "host".
 *  - `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream, never
 *    synchronises, never allocates (callers pass workspaces; heal_*_workspace() gives the size).
 *  - return value: 0 on success, negative HEAL_ERR_* otherwise (no exceptions cross the ABI).
 *  - activations are channels-last: a (N,C,H,W) map is stored as [n][h][w][c]; `cstride` is the
 *    distance in floats between two pixels and `coffset` the first channel used, so that a conv can
 *    read / write a channel slice of a wider concat buffer.
 */
#ifndef HEAL_B200_H_
#define HEAL_B200_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HEAL_B200_ABI_VERSION 3

/* Activation tensor view (channels-last).  fmt: 0 = fp32, 1 = bf16 (one plane), 2 = split-bf16
 * (hi = bf16(x) at data, lo = bf16(x-hi) at data + plane_stride elements; x ~ hi+lo, 16 mantissa bits).
 * cstride = elements between consecutive pixels, coffset = first channel used.
 * Split holds finite values only: +-inf stored as split loads back as NaN (hi = inf, lo = bf16(inf - inf) = NaN). */
#define HEAL_FMT_F32 0
#define HEAL_FMT_BF16 1
#define HEAL_FMT_SPLIT 2
typedef struct {
    void* data;
    int fmt;
    int cstride;
    int coffset;
    size_t plane_stride;
} heal_act_t;
int heal_abi_version(void);
/* sm_90a build check: returns 0 when a Hopper (cc 9.x) device is current, negative otherwise. */
int heal_device_check(void);
/* number of kernels this library has launched in this process so far */
long long heal_launch_count(void);

/* ---- voxelization -------------------------------------------------------------------------
 * replaces SpVoxelPreprocessor.preprocess + collate_batch for all agents of a scene
 * (opencood/data_utils/pre_processor/sp_voxel_preprocessor.py:62-85, :145-174 -> spconv CPU
 * VoxelGeneratorV2.generate / Point2VoxelCPU3d.point_to_voxel). Bit-exact: voxel order = order of
 * first appearance, first `max_points_per_voxel` points in input order, cells beyond `max_voxels`
 * dropped, coords = [agent, z, y, x].
 *   points          (P_total,4) f32, agents concatenated
 *   agent_offsets   (A+1) i32 device: points of agent a are [off[a], off[a+1]); rows before off[0] and from off[A] on
 *                   are ignored
 *   range_min3/voxel_size3/grid3   HOST arrays (x,y,z)
 *   capacity        rows available in the outputs; voxel rows >= capacity are dropped (nothing is written past it)
 *   voxels_out      (capacity,T,4) f32   coords_out (capacity,4) i32   num_points_out (capacity) i32
 *   num_voxels_out  (1+A) i32: [0] = M total, [1+a] = voxels of agent a, counted before the capacity cut, so
 *                   min(M, capacity) rows are valid */
size_t heal_voxelize_workspace(int num_points_total, int capacity, int num_agents);
int heal_voxelize(const float* points, const int* agent_offsets, int num_agents, int num_points_total,
                  const float* range_min3_host, const float* voxel_size3_host, const int* grid3_host,
                  int max_points_per_voxel, int max_voxels, int capacity,
                  float* voxels_out, int* coords_out, int* num_points_out, int* num_voxels_out,
                  void* workspace, size_t workspace_bytes, void* stream);

/* MeanVFE.forward (opencood/models/sub_modules/mean_vfe.py:13-33): (M,T,4) -> (M,4) */
int heal_mean_vfe(const float* voxels, const int* num_points, int num_voxels, int max_points_per_voxel,
                  float* mean_out, void* stream);

/* ---- PillarVFE + PointPillarScatter, fused --------------------------------------------------
 * replaces PillarVFE.forward (opencood/models/sub_modules/pillar_vfe.py:105-155, PFNLayer :31-53)
 * and PointPillarScatter.forward (opencood/models/sub_modules/point_pillar_scatter.py:19-77).
 *   w_folded (10,64) = linear.weight^T * bn_scale, b_folded (64) = bn_shift (folded on the host, fp64)
 *   offset3_host = voxel_size/2 + range_min (x,y,z)
 *   pillar_features_out (M,64) fp32 or NULL; pillar_split_rows_out (M,128) bf16 [hi 64 | lo 64] or NULL (the gather source of
 *   the tensor-core sparse stem); canvas_out: (B,ny,nx,64) channels-last view in any storage
 *   format, pre-zeroed by the caller, or NULL
 *   num_voxels_dev: optional device count (row 0 used) so a graph-captured frame needs no host sync */
int heal_pillar_vfe_scatter(const float* voxel_features, const int* voxel_num_points, const int* voxel_coords,
                            const int* num_voxels_dev, int num_voxels, int max_points_per_voxel,
                            const float* w_folded, const float* b_folded, int c_in, int c_out,
                            const float* voxel_size3_host, const float* offset3_host, int nx, int ny,
                            float* pillar_features_out, void* pillar_split_rows_out, const heal_act_t* canvas_out, void* stream);

/* Stand-alone PointPillarScatter.forward (opencood/models/sub_modules/point_pillar_scatter.py:19-77): rows of pillar features
 * (M,channels) f32 -> canvas cell [b][y][x + z] of a pre-zeroed channels-last canvas view (any storage format). */
int heal_pillar_scatter(const float* pillar_features, const int* voxel_coords, const int* num_voxels_dev, int num_voxels,
                        int channels, int nx, int ny, const heal_act_t* canvas_out, void* stream);

/* ---- sparse stem: scatter + the first residual block's two stride-2 convs straight from the pillar list -------------
 * heal_pillar_idmap: (B,ny,nx) i32 map, cell -> pillar row or -1 (replaces the dense canvas of PointPillarScatter,
 * point_pillar_scatter.py:19-77, as the conv input).
 * heal_sparse_stem: out_conv = ReLU(bn1(conv1 3x3 stride 2 pad 1 (canvas))), out_down = bn(downsample 1x1 stride 2 (canvas))
 * (BasicBlock, resblock.py:48-64 with the downsample of :178-187) for 64 -> 64 channels; w_conv3x3 fp32 [9][64][64]
 * (tap, cin, cout), w_down1x1 fp32 [64][64] (cin, cout), BN folded; outputs (B, ny/2, nx/2, 64) in any storage format. */
int heal_pillar_idmap(const int* voxel_coords, const int* num_voxels_dev, int num_voxels, int batch, int ny, int nx,
                      int* idmap_out, void* stream);
int heal_sparse_stem(const float* pillar_features, const int* idmap, int batch, int ny, int nx,
                     const float* w_conv3x3, const float* b_conv3x3, const float* w_down1x1, const float* b_down1x1,
                     int channels, const heal_act_t* out_conv, const heal_act_t* out_down, void* stream);
/* Same contract on the tensor cores (mma.sync m16n8k16, split-bf16 hi/lo operands: fp32-equivalent, ~1e-6 relative, not
 * bit-identical to the fp32 FMA order); needs nx % 32 == 0.  A warp owns 16 output pixels, all ten weight matrices stay in smem. */
int heal_sparse_stem_tc(const float* pillar_features, const int* idmap, int batch, int ny, int nx,
                        const float* w_conv3x3, const float* b_conv3x3, const float* w_down1x1, const float* b_down1x1,
                        int channels, const heal_act_t* out_conv, const heal_act_t* out_down, void* stream);

/* ---- 2-D convolution, fp32 CUDA-core path ---------------------------------------------------
 * replaces nn.Conv2d / nn.ConvTranspose2d(k==stride) + eval BatchNorm2d + ReLU (+ residual add) of
 * resblock.py:48-64,102-122, base_bev_backbone.py:40-86, base_bev_backbone_resnet.py:54-85,
 * downsample_conv.py:16-27, heter_pyramid_collab.py:102-107.  fp32 FMA math whatever the storage
 * format of in / residual / out (heal_act_t).
 *   weight: groups==1 : fp32 [kh][kw][Cin][w_cstride] (w_cstride >= Cout, multiple of 4), BN scale folded
 *           groups>1  : fp32 [kh*kw][Cin/groups][Cout/groups][groups] (3x3 only, Cin==Cout)
 *   output pixel (oh,ow) of the (Ho,Wo) conv grid is stored at (oh*upsample+up_i, ow*upsample+up_j)
 *   of an (Ho*upsample, Wo*upsample) map: a k==stride transposed conv is upsample^2 1x1 launches.
 *   in is read 4 channels at a time: Cin, in->cstride, in->coffset (and the split plane stride) multiples of 4 and in->data
 *   16-byte aligned (fp32) or 8-byte aligned (bf16 / split), else HEAL_ERR_UNSUPPORTED.  The grouped conv writes 4 channels
 *   at a time and refuses an out view that fails the same rule; the dense conv writes such a view one channel at a time. */
int heal_conv2d_simt(const heal_act_t* in, int N, int H, int W, int Cin,
                     const float* weight, int w_cstride, const float* bias,
                     int kh, int kw, int stride, int pad, int groups,
                     const heal_act_t* residual, const heal_act_t* out, int Ho, int Wo, int Cout,
                     int upsample, int up_i, int up_j, int relu, void* stream);

/* ---- 2-D convolution, wgmma tensor-core path ---------------------------------------------------
 * Same reference ops as heal_conv2d_simt, evaluated as an implicit GEMM with wgmma (register
 * accumulators) fed by TMA.  Activations are "split-bf16": `planes` bf16 channels-last planes
 * (planes=2: hi = bf16(x), lo = bf16(x-hi), fp32-equivalent via the three products a_hi*b_hi + a_hi*b_lo + a_lo*b_hi per K
 * step; planes=1: plain bf16).
 *   in_split   bf16 [planes][N][H][W][in_cstride], plane stride in elements; Cin % 64 == 0
 *   w_packed   bf16 [planes][w_rows][Cin]; conv: w_rows = kh*kw*coutp, row = tap*coutp + co;
 *              transposed conv (kh=kw=1, upsample=k): w_rows = k*k*coutp, row = (i*k+j)*coutp + co;
 *              coutp = Cout padded to 16/32/64 or a multiple of 128; BN scale folded; bias fp32 [Cout]
 *   residual   split planes (res_split) or fp32 (res_f32) or neither, at output resolution
 *   outputs    split planes and/or fp32, channels-last, output map (Ho*upsample, Wo*upsample)
 *   stride     1 or 2 (TMA element strides on W/H)
 *   blockdiag  1: grouped 3x3 conv (Cin == Cout == coutp, channels-per-group | 64) evaluated as block-diagonal
 *              64x64 channel blocks; w_packed is then [planes][kh*kw*coutp][64] (row = tap*coutp + co,
 *              column = input channel within co's 64-channel block, zeros outside co's group);
 *              w_diag (optional, NULL otherwise): the same weights as [planes][kh*kw][coutp][16] — only the 16x16 diagonal
 *              sub-block of each output channel; when given, the kernel streams these (a quarter of the bytes, 32 B-swizzled
 *              TMA boxes) instead of the 64-wide rows of w_packed */
/* planes / w_planes of heal_conv2d_tc: activation planes (1 = bf16, 2 = split-bf16) and weight planes. (2,2) = fp32-equivalent
 * "tc32"; (1,2) = the "bf16" engine mode: bf16 activations x split (un-rounded) weights, a_hi x [b_hi | b_lo]; (1,1) = plain bf16. */
int heal_conv2d_tc(const void* in_split, size_t in_plane_stride, int N, int H, int W, int Cin, int in_cstride, int in_coffset,
                   const void* w_packed, const void* w_diag, int w_rows, int coutp, const float* bias,
                   int kh, int kw, int stride, int pad, int blockdiag, int planes, int w_planes,
                   const void* res_split, size_t res_plane_stride, const float* res_f32, int res_cstride, int res_coffset,
                   void* out_split, size_t out_plane_stride, int out_cstride, int out_coffset,
                   float* out_f32, int out32_cstride, int out32_coffset,
                   int Ho, int Wo, int Cout, int upsample, int relu, void* stream);

/* ---- 3x3 convolution of a narrow input, wgmma tensor-core path -----------------------------------
 * out = act(conv3x3(in) + bias), stride 1, pad 1, groups 1, for 1 <= Cin <= 63 (NaiveCompressor's first decoder conv: the
 * compressed map is narrower than heal_conv2d_tc's 64-channel K blocks).  The implicit GEMM's K is the whole neighbourhood:
 * k = tap * cinp + ci with tap = ky * 3 + kx, cinp = Cin rounded up to even, K = 9 * cinp rounded up to a multiple of 16.
 *   in         any storage format (f32, bf16, split), any channel stride >= coffset + Cin (a channel slice is fine)
 *   w_packed   bf16 [ceil(Cout / 64)][ceil(K / 64)][128][64], 16-byte aligned: per 64-channel output block and 64-wide K block,
 *              rows 0..63 = hi = bf16(w) and rows 64..127 = lo = bf16(w - hi) of output channels 64 * block + row, column = k;
 *              zero in the pad channel of an odd Cin, for k >= 9 * cinp and for channels >= Cout; BN scale folded
 *   bias       fp32 [Cout] (folded BN shift), 8-byte aligned
 *   planes     2: split-bf16 activations, a_hi*b_lo + a_lo*b_hi + a_hi*b_hi per K step (fp32-equivalent, "tc32");
 *              1: bf16 activations, a_hi*b_lo + a_hi*b_hi ("bf16").  The input is read as fp32 and split by the kernel.
 *   relu       0 | 1
 *   out        (N,H,W,Cout) in any storage format; channel stride, offset and plane stride even, data 8-byte (f32) or
 *              4-byte (bf16, split) aligned, else HEAL_ERR_UNSUPPORTED.
 * Cout is a multiple of 16 in [16, 256].  Allocates nothing and does not synchronise. */
int heal_conv3x3_narrow_tc(const heal_act_t* in, int N, int H, int W, int Cin, const void* w_packed, const float* bias,
                           int Cout, int planes, int relu, const heal_act_t* out, void* stream);

/* ---- ResNeXt bottleneck, fused (PyramidFusion level 0) ------------------------------------------
 * y = ReLU(conv3(ReLU(conv2(ReLU(conv1(x))))) + x) for the stride-1 Bottleneck with C = 64 input / output channels, width 128,
 * 32 groups and no downsample (BN folded into each conv), as one kernel: the width-128 intermediates stay on chip.  The three
 * weights are the packings heal_conv2d_tc takes for those convs (w_planes = 2): w1 [2][128][64], w2_diag [2][9*128][16] (the
 * diagonal sub-blocks of the grouped conv), w3 [2][64][128]; biases fp32.  planes 2 (split-bf16) or 1 (bf16).  The output is
 * bit-identical to the three heal_conv2d_tc launches and may be a channel slice [out_coffset, out_coffset + 64) of a wider map. */
int heal_bottleneck_tc(const void* x, size_t x_plane_stride, int N, int H, int W, int C, int x_cstride,
                       const void* w1, const float* b1, const void* w2_diag, const float* b2, const void* w3, const float* b3,
                       int planes, int w_planes, void* out, size_t out_plane_stride, int out_cstride, int out_coffset, void* stream);

/* ---- ResNeXt bottleneck, grouped 3x3 + 1x1 reduce fused (PyramidFusion levels 1 and 2) -------------
 * y = ReLU(conv3(ReLU(conv2(mid))) + res) for the stride-1 Bottleneck's grouped 3x3 (32 groups, width channels) and 1x1 reduce
 * (width -> Cout) with the identity residual, as one kernel: the grouped conv's output stays on chip.  mid is the expand's
 * output (N,H,W,width), res the block input (N,H,W,Cout).  The weights are the packings heal_conv2d_tc takes for those convs
 * (w_planes = 2): w2_diag [2][9*width][16] (the diagonal sub-blocks of the grouped conv), w3 [2][Cout][width]; biases fp32.
 * width a multiple of 64, Cout a multiple of 128; planes 2 (split-bf16) or 1 (bf16).  The output is bit-identical to the two
 * heal_conv2d_tc launches and may be a channel slice [out_coffset, out_coffset + Cout) of a wider map. */
int heal_gconv_reduce_tc(const void* mid, size_t mid_plane_stride, int N, int H, int W, int width, int mid_cstride,
                         const void* w2_diag, const float* b2, const void* w3, const float* b3, int Cout,
                         const void* res, size_t res_plane_stride, int res_cstride, int planes, int w_planes,
                         void* out, size_t out_plane_stride, int out_cstride, int out_coffset, void* stream);

/* ---- PyramidFusion weighted fuse of one level -------------------------------------------------
 * replaces weighted_fuse (opencood/models/fuse_modules/pyramid_fuse.py:17-63) incl. both
 * warp_affine_simple calls (torch_transformation_utils.py:323-332), score = sigmoid(occ)+1e-4
 * (:145) and the eval-mode camera crop mask (:147-162) for ONE scene.
 *   feat (n,H,W,C) channels-last; occ (n,H,W) logits; theta (n,2,3) f64 = affine_matrix[b,0,:n]
 *   crop_windows (n,4) i32 [h0,h1,w0,w1] (score kept inside, zeroed outside) or NULL
 *   agent_feat_offsets_host / agent_occ_offsets_host: HOST arrays of n element offsets of agent j's feature map (from
 *     feat->data, in elements of the storage type) and occupancy map (from occ, in floats); NULL = dense stacks
 *     (j*H*W*cstride, j*H*W).  This is how the kernel reads the agents straight out of the all-gathered buffer of the
 *     agent-per-GPU partition (SURVEY.md 8e) without an unpack copy.
 *   row0, rows: produce output rows [row0, row0+rows) only (row-sharded fusion tail); rows <= 0 = the whole map
 *   out (rows,W,C): the output slab, its pixel 0 is (row0, 0)
 * Alignment: C, the channel strides and offsets of feat and out, their plane strides and the agent feature offsets are
 * multiples of 4 elements, and feat->data / out->data are 16-byte aligned for fp32 and 8-byte aligned for bf16 / split;
 * anything else returns HEAL_ERR_UNSUPPORTED.  Split input takes the 8-channel kernel only when C, its strides, offsets and
 * agent offsets are multiples of 8 and feat->data is 16-byte aligned, the generic kernel otherwise (same results). */
int heal_pyramid_fuse_level(const heal_act_t* feat, const float* occ, const double* theta,
                            const int* crop_windows, int n_agents, int H, int W, int C, int align_corners,
                            const long long* agent_feat_offsets_host, const long long* agent_occ_offsets_host,
                            int row0, int rows, const heal_act_t* out, void* stream);

/* AttFusion.forward for one scene (opencood/models/fuse_modules/fusion_in_one.py:126-151).  C in {128, 256, 384, 512},
 * n_agents <= 8.  Alignment as heal_pyramid_fuse_level: strides, offsets and plane strides multiples of 4 elements, data
 * 16-byte aligned (fp32) or 8-byte aligned (bf16 / split), else HEAL_ERR_UNSUPPORTED; split input with C <= 256, strides and
 * offsets multiples of 8 and a 16-byte aligned data pointer takes the 8-channel kernel.  C = 64 (the first level of
 * HeterModelBaselineMs) takes its own kernel, for every input format, with 16-byte loads and stores: input and output data
 * 16-byte aligned and, for bf16 / split, strides, offsets and plane strides multiples of 8 (fp32: of 4), else
 * HEAL_ERR_UNSUPPORTED. */
int heal_att_fuse(const heal_act_t* feat, const double* theta, int n_agents, int H, int W, int C,
                  const heal_act_t* out, void* stream);

/* MaxFusion.forward for one scene (fusion_in_one.py:87-124): out(H,W,C) = max over j of warp(feat_j, theta[j]).
 * Pixels warped in from outside agent j's map are 0 and take part in the max.  feat (n,H,W,C), theta (n,2,3) fp64 device;
 * C, channel strides, offsets and plane strides multiples of 4; feat->data / out->data 16-byte aligned for fp32, 8-byte
 * aligned for bf16 / split (else HEAL_ERR_UNSUPPORTED). */
int heal_max_fuse(const heal_act_t* feat, const double* theta, int n_agents, int H, int W, int C,
                  const heal_act_t* out, void* stream);

/* A batch of warp_affine_simple (bilinear, zeros padding, align_corners=False):
 * out image k = grid_sample(src image src_index_host[k], theta[k]) for k < n_out.
 * src_index_host: HOST array of n_out image indices into src (H,W,C maps); theta (n_out,2,3) fp64 device; out (n_out,H,W,C).
 * Alignment of src and out as heal_max_fuse. */
int heal_warp_affine(const heal_act_t* src, const int* src_index_host, const double* theta, int n_out,
                     int H, int W, int C, const heal_act_t* out, void* stream);

/* V2VNet message aggregation (fusion_in_one.py:262-300) for n_nodes updated nodes.  nodes_host: HOST array of n_nodes
 * int quadruples (x image, P image, first pair row r, neighbours n).  For updated node u and j < n:
 *   msg_j = mask_j * (q[r + j] + p_node[P image]),  mask_j = warp(ones, theta[r + j]) (recomputed from the taps)
 *   agg   = mean_j msg_j (agg_max = 0, divides by n) or max_j msg_j (agg_max = 1)
 * gru = 1: out image u (2C channels) = [x | agg]  (the ConvGRU input);  gru = 0: out image u (C channels) = x + agg.
 * q (pairs,H,W,C) = W[:, :C] (*) warped neighbours; p_node (.,H,W,C) = W[:, C:] (*) x + bias; theta (pairs,2,3) fp64 device.
 * Alignment of q, p_node, x and out as heal_max_fuse. */
int heal_v2v_aggregate(const heal_act_t* q, const heal_act_t* p_node, const heal_act_t* x, const double* theta,
                       const int* nodes_host, int n_nodes, int H, int W, int C, int agg_max, int gru,
                       const heal_act_t* out, void* stream);

/* Where2commFusion's attention core (fusion_in_one.py:431-484; where2comm_attn.py EncodeLayer.attn, an 8-head
 * nn.MultiheadAttention): per scene b, pixel and head, one query (the warped ego) over the scene's n_b agents warped to it.
 *   q    (B, H, W, C): the in-projected warped ego, bias included, not yet scaled
 *   kv   (sum n_b, H, W, 2C): [W_k; W_v] x_j of the UNWARPED agent maps, bias-free, in record_len order (each scene's ego
 *        first); a channel view of a wider map is fine
 *   kv_bias: (2C) fp32 device, 16-byte aligned: [b_k; b_v], added after sampling
 *   theta (sum n_b, 2, 3) fp64 device: affine[b, 0, j] stacked scene by scene
 *   out  (B, H, W, C): the merged heads, before out_proj
 * k_j = warp(kv_j, theta_j)[:C] + b_k and v_j = warp(kv_j, theta_j)[C:] + b_v (bilinear, zeros padding, align_corners=False:
 * the taps of heal_att_fuse; a linear map commutes with the warp, so this is the projection of the warped map).  Per head:
 * out = sum_j softmax_j((q * dim_head^-0.5) . k_j) v_j, the scale applied to q in fp32 as PyTorch does, the max subtracted
 * before the exponent, agents summed in order; fp32 math for every storage format, no atomics (bit-identical reruns).
 * C = 256 and heads = 8 (dim_head 32), else HEAL_ERR_UNSUPPORTED.  n_agents_host: HOST array of B counts in [1, 8], all checked
 * before anything is launched (else HEAL_ERR_ARG).  Alignment of q, kv and out as heal_max_fuse. */
int heal_ego_mha(const heal_act_t* q, const heal_act_t* kv, const float* kv_bias, const double* theta,
                 const int* n_agents_host, int B, int H, int W, int C, int heads, const heal_act_t* out, void* stream);

/* ConvGRU cell with a zero hidden state (sub_modules/convgru.py:47-68): out(npix,C) = sigmoid(zc[:, :C]) * tanh(zc[:, C:2C]),
 * zc = the stacked (update gate | candidate) GRU conv output (npix, 2C).  Alignment of zc and out as heal_max_fuse. */
int heal_gru_gate(const heal_act_t* zc, long long npix, int C, const heal_act_t* out, void* stream);

/* CoBEVT window / grid attention core (swap_fusion_modules.py:87-128 with CoBEVT's agent mask, fusion_in_one.py:409-429).
 * qkv (B*L, H, W, 3C) = the to_qkv 1x1-conv output (q | k | v, head h = channels h*32 .. h*32+31 of each; q already scaled by
 * 32^-0.5); out (B*L, H, W, C) = the merged heads.  One window has n = L*w*w tokens ordered (agent l, w1, w2):
 *   grid_mode 0 (window):  window (x, y) = pixels (x*w + w1, y*w + w2)
 *   grid_mode 1 (grid):    window (x, y) = pixels (w1*H/w + x, w2*W/w + y)
 * out_i = sum_j softmax_j(q_i . k_j + bias[h][j][i]) v_j over the keys of the n_agents_host[b] real agents of scene b (tokens
 * j < n_agents_host[b]*w*w); the keys of padded agents are skipped (the reference's -inf), their queries are computed.
 * bias: (C/32, n, n) fp32 device, KEY-major: bias[h][j][i] = relative_position_bias_table[relative_position_index[i][j]][h].
 * n_agents_host: HOST array of B counts in [1, L].  C a multiple of 32 (dim_head 32), n <= 128, H and W multiples of w. */
int heal_swap_attention(const heal_act_t* qkv, const int* n_agents_host, int B, int L, int H, int W, int C,
                        int window_size, int grid_mode, const float* bias, const heal_act_t* out, void* stream);

/* Mean over n_avg consecutive images, then LayerNorm over the channels (biased variance, eps):
 * out image o = LayerNorm(mean_{k < n_avg} in image o*n_avg + k) for o < n_out.  n_avg = 1 is a plain LayerNorm.
 * ln_weight, ln_bias: (C) fp32 device.  C in {64, 128, 192, 256}.  n_out = 0 launches nothing (in / out data may be NULL). */
int heal_mean_layernorm(const heal_act_t* in, int n_out, int n_avg, int H, int W, int C, const float* ln_weight,
                        const float* ln_bias, float eps, const heal_act_t* out, void* stream);

/* ---- V2X-ViT (fusion_in_one.py:320-372, sub_modules/v2xvit_basic.py) ---------------------------
 * One BaseWindowAttention branch (mswin.py:20-92): softmax(q k^T + bias) v over the w x w windows of every image, on the
 * tensor cores.  qkv (n_img, H, W, 3*heads*dim_head) = the branch's to_qkv 1x1-conv output from the view's coffset
 * (q | k | v, head m = channels m*dim_head .. of each; q already scaled by dim_head^-0.5); out (n_img, H, W, heads*dim_head)
 * = the merged heads, at the view's coffset (a channel slice of a wider map is fine).  Window (x, y) holds pixels
 * (x*w + w1, y*w + w2), token t = w1*w + w2.  bias: (w^2, w^2) fp32 device, query-major, shared by every head and window.
 * bf16 storage: bf16 operands, fp32 accumulation; fp32 and split-bf16 storage: split-bf16 products (fp32-equivalent).
 * window_size in {4, 8, 16}, dim_head in {16, 32, 64}, H and W multiples of window_size; bias 8-byte aligned, data pointers,
 * channel offsets and strides of qkv / out even (pairs of channels are read and written together). */
int heal_window_attention(const heal_act_t* qkv, int n_img, int H, int W, int heads, int dim_head, int window_size,
                          const float* bias, const heal_act_t* out, void* stream);

/* The per-pixel HGTCavAttention core (hmsa.py) with every agent of type 0: for each query agent i, head and pixel,
 * softmax_j(q_i . k_j) over the n_b real agents of its scene, then sum_j p_j v_j.  qkv (N, H, W, 3C) = q | k | v of the
 * folded to_qkv conv (relation_att[0] and dim_head^-0.5 folded into q, relation_msg[0] into v), dim_head 32.  Image layout:
 * the ego of scene b is image b (b < B); its other n_b - 1 agents follow at image B + sum_{b' < b} (n_b' - 1).  ego_only 0:
 * out has the N images of qkv; ego_only 1: out (B, H, W, C) holds the egos' outputs only.  n_agents_host: HOST array of B
 * counts in [1, 8], all checked before anything is launched. */
int heal_cav_attention(const heal_act_t* qkv, const int* n_agents_host, int B, int H, int W, int C, int ego_only,
                       const heal_act_t* out, void* stream);

/* SplitAttn (split_attn.py) with the PreNorm residual: o (n_img, H, W, 3C) = the three to_out outputs side by side, x the
 * residual.  gate = softmax over the 3 branches of fc2(ReLU(LayerNorm(fc1(mean_{H,W}(o_0 + o_1 + o_2))))) per image and
 * channel; out = o_0 * g_0 + o_1 * g_1 + o_2 * g_2 + x (out may be x).  fc1_t (C, C) and fc2_t (C, 3C) fp32 device, the
 * Linear weights transposed (fc1_t[k][c] = fc1.weight[c][k]).  The pooled sum is reduced in a fixed order (no atomics).
 * C = 256.  workspace: heal_split_attn_workspace(n_img, C) bytes of device memory, 16-byte aligned. */
size_t heal_split_attn_workspace(int n_img, int C);
int heal_split_attn(const heal_act_t* o, const heal_act_t* x, int n_img, int H, int W, int C, const float* fc1_t,
                    const float* ln_w, const float* ln_b, float eps, const float* fc2_t, void* workspace, size_t ws_bytes,
                    const heal_act_t* out, void* stream);

/* The STTF resample (v2xvit_basic.py:12-33, torch_transformation_utils.warp_affine): out image k = F.grid_sample(src image k,
 * F.affine_grid(theta[k], align_corners=True)), bilinear, zeros padding, align_corners=True.  theta: (n_img, 2, 3) fp32
 * device.  C a multiple of 4. */
int heal_sttf_resample(const heal_act_t* src, const float* theta, int n_img, int H, int W, int C, const heal_act_t* out,
                       void* stream);

/* ---- Lift-Splat-Shoot ------------------------------------------------------------------------
 * heal_lss_cell_index replaces LiftSplatShoot.get_geometry + the index half of voxel_pooling
 * (opencood/models/heter_encoders.py:125-147, :173-185): for every frustum point of every camera image
 * the BEV cell (z*ny + y)*nx + x, or -1 when outside the grid (`.long()` truncation kept).
 *   frustum (D,fH,fW,3) f32; post_rots_inv / combine (BN,3,3) = inverse(post_rots), rots@inverse(intrins)
 *   (tiny 3x3 algebra done by the caller exactly as the reference does); post_trans / trans (BN,3)
 *   lower3 = bx - dx/2, dx3, nx3: HOST arrays (x,y,z) in the reference's fp32 values
 * heal_lss_pool replaces CamEncode's depth softmax (x) feature outer product
 * (opencood/models/sub_modules/lss_submodule.py:132-134, :227-229) and voxel_pooling's per-cell sum
 * (heter_encoders.py:188-212): bev_out (agents, nz*ny*nx, C) channels-last fp32, pre-zeroed (nz == 1 gives
 * the reference's (B,C,ny,nx) map). depth_logits (BN,D,fH,fW), feat (BN,C,fH,fW) as the torch heads emit them. */
/* per-camera 3x3 algebra of get_geometry (heter_encoders.py:135,142), capturable in a CUDA graph (torch.inverse is not):
 * post_rots_inv_out = inverse(post_rots), combine_out = rots @ inverse(intrins); all (num_images,3,3) f32 row-major, device. */
int heal_lss_camera_matrices(const float* rots, const float* intrins, const float* post_rots, int num_images,
                             float* post_rots_inv_out, float* combine_out, void* stream);
int heal_lss_cell_index(const float* frustum, int D, int fH, int fW,
                        const float* post_rots_inv, const float* post_trans, const float* combine, const float* trans,
                        int num_images, const float* lower3_host, const float* dx3_host, const int* nx3_host,
                        int* cell_out, void* stream);
int heal_lss_pool(const float* depth_logits, const float* feat, const int* cell, int num_images, int cams_per_agent,
                  int D, int C, int fH, int fW, int cells_per_agent, float* bev_out, void* stream);

/* Deterministic variant of heal_lss_pool (the default path): cell-sorted interval reduction, no atomics.  Points are radix-sorted
 * (stable, CUB) by agent*cells + cell; the sorted list is cut into equal chunks of 128 points (one block each, thread = channel):
 * cells inside a chunk are summed in ascending point order and written directly, cells crossing chunk boundaries are combined
 * from per-chunk partial sums in chunk order -- a fixed summation order, every run gives the same bits (the reference's
 * QuickCumsum, opencood/utils/camera_utils.py:220-246, is likewise a sum over a sorted interval).  bev_out must be PRE-ZEROED
 * (cells no frustum point falls into are not written).
 *   depth_logits / feat with ELEMENT strides (image, depth-bin | channel, pixel): NCHW torch tensors (HW*D, HW, 1) or the
 *   channels-last output of the fused 1x1 heads (HW*S, 1, S).  bev_out: (agents, cells_per_agent, C) channels-last view, any format. */
size_t heal_lss_pool_sorted_workspace(int num_images, int D, int fH, int fW, int agents, int cells_per_agent);
int heal_lss_pool_sorted(const float* depth_logits, long long l_img, long long l_d, long long l_pix,
                         const float* feat, long long f_img, long long f_c, long long f_pix,
                         const int* cell, int num_images, int cams_per_agent, int D, int C, int fH, int fW,
                         int cells_per_agent, const heal_act_t* bev_out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- sparse 3-D convolution (SECOND VoxelBackBone8x) + HeightCompression ------------------------
 * Replaces the spconv calls of opencood/models/sub_modules/sparse_backbone_3d.py:48-91,:114-130 and
 * height_compression.py:21-23.  A sparse tensor = feats (rows,C) f32 + coords (rows,4) i32 [b,z,y,x] + a device
 * row count; `*_capacity` bounds the rows, `*_rows_dev` (nullable) is the live count.  A hash table
 * (keys u32, vals i32, heal_spconv_table_size(capacity) entries each) maps a site to its row.
 * Rulebooks are output-stationary: nbr[row][k] = input row under kernel offset k (z-major, then y, x) or -1.
 *  - build_table          site -> row map of an existing tensor (first level, from the voxelizer's coords)
 *  - subm_neighbors       SubMConv3d rulebook (output sites = input sites), shared by every conv with the same indice_key;
 *                         table_capacity = the capacity the table was built with (its size = heal_spconv_table_size of it)
 *  - strided_rulebook     SparseConv3d: output sites (deterministic order), their table, and the rulebook
 *  - gather_gemm          out[r] = act(bias + sum_k in[nbr[r][k]] . W[k]),  W fp32 [kvol][Cin][Cout] with BN folded
 *  - sparse_to_bev        .dense() + view(N, C*D, H, W): bev_out (B,H,W,C*D) channels-last fp32, pre-zeroed, channel = c*D+z */
size_t heal_spconv_table_size(int capacity);
int heal_spconv_build_table(const int* coords, const int* num_rows_dev, int capacity, const int* spatial_shape3_host, int batch,
                            uint32_t* table_keys, int* table_vals, void* stream);
int heal_spconv_subm_neighbors(const int* coords, const int* num_rows_dev, int capacity, const int* spatial_shape3_host,
                               const int* ksize3_host, const uint32_t* table_keys, const int* table_vals, int table_capacity,
                               int* nbr_out, void* stream);
size_t heal_spconv_strided_workspace(int in_capacity, int out_capacity, int kvol);
int heal_spconv_strided_rulebook(const int* in_coords, const int* in_rows_dev, int in_capacity,
                                 const int* out_spatial_shape3_host, int batch,
                                 const int* ksize3_host, const int* stride3_host, const int* pad3_host,
                                 int out_capacity, int* out_coords, int* out_rows_dev,
                                 uint32_t* out_table_keys, int* out_table_vals, int* nbr_out,
                                 void* workspace, size_t workspace_bytes, void* stream);
int heal_spconv_gather_gemm(const float* in_feats, const int* nbr, const int* out_rows_dev, int out_capacity, int kvol,
                            const float* weight, const float* bias, int c_in, int c_out, int relu,
                            float* out_feats, void* stream);

/* The same gather-GEMM on the tensor cores (csrc/spconv_tc.cu: wgmma, register accumulators, cp.async row gather into
 * 128B-swizzled K-major tiles, TMA weight tiles), for c_in in {16,32,64}.  Features are "split rows": (rows, 2*C) bf16 =
 * [hi C | lo C] with x ~= hi + lo; products a_hi*b_hi + a_hi*b_lo + a_lo*b_hi, fp32 accumulation (fp32-equivalent).
 *   w_packed   [2 planes][KB * c_out rows][64] bf16, KB = ceil(kvol / (64 / c_in)); column = (offset within K-block) * c_in + ci
 *   out_split_rows (capacity, 2*c_out) bf16 and / or out_f32 (capacity, c_out)
 *   in_pitch / in_lo / out_pitch / out_lo (elements; 0 = the interleaved-row defaults 2C / C): row pitch and hi->lo distance, so
 *   that the kernel can also gather from / write to a PLANAR split activation (pitch = pixel stride, lo = plane stride) -- used
 *   by the PointPillars sparse stem, whose outputs are dense BEV maps in the conv engine's format. */
int heal_spconv_gather_gemm_tc(const void* in_split_rows, const int* nbr, const int* out_rows_dev, int out_capacity, int kvol,
                               const void* w_packed, const float* bias, int c_in, int c_out, int relu,
                               void* out_split_rows, float* out_f32,
                               long long in_pitch, long long in_lo, long long out_pitch, long long out_lo, void* stream);
/* Rulebook of a ksize x ksize / stride-2 2-D convolution from the pillar list to the dense (batch, ny/2, nx/2) output grid:
 * nbr_out[(b*Ho + oy)*Wo + ox][r*ksize + s] = idmap[b][2oy + r - pad][2ox + s - pad] or -1 (idmap: heal_pillar_idmap). */
int heal_stem_rulebook(const int* idmap, int batch, int ny, int nx, int ksize, int pad, int* nbr_out, void* stream);
/* fp32 rows (capacity, C) -> split rows (capacity, 2*C) bf16 */
int heal_rows_to_split(const float* rows_f32, const int* rows_dev, int capacity, int channels, void* out_split_rows, void* stream);
int heal_sparse_to_bev(const float* feats, const int* coords, const int* rows_dev, int capacity, int C, int D, int H, int W,
                       float* bev_out, void* stream);

/* ---- detection post-processing (SURVEY 8f rank 1) ---------------------------------------------------------------
 * replaces VoxelPostprocessor.post_process for one cav (voxel_postprocessor.py:245-405): sigmoid + score threshold,
 * delta_to_boxes3d (:408-453), direction-bin fix (:314-330), boxes_to_corners_3d + project_box3d (box_utils.py:152-204, 278-316),
 * remove_large_pred_bbx / remove_bbx_abnormal_z (:840-890), nms_rotated on the `top` best scores (:693-738, polygon IoU in
 * fp64), mask_boxes_outside_range_numpy (:384-421).  Everything stays on the device and on the caller's stream.
 *   cls (1,H,W,A) logits, reg (1,H,W,7A) deltas, dir (1,H,W,A*num_bins) or NULL: fp32 channels-last views (heal_act_t fmt 0)
 *   anchors: device fp32 (H,W,A,7) [x y z h w l yaw] ('hwl' order, order_hwl = 1) or [x y z l w h yaw]
 *   transform4x4_host: row-major cav -> ego matrix; range6_host: [minx miny minz maxx maxy maxz] or NULL (no range mask).  A box
 *     is kept when every corner c has lo <= c <= hi in fp32.  The reference compares fp32 corners with float64 limits, so callers
 *     pass each lower limit rounded up to the smallest fp32 >= it and each upper limit rounded down to the largest fp32 <= it
 *     (ops._box_range_f32); the fp32 test is then exactly the float64 one (a corner at float32(-25.6) < -25.6 is dropped).
 *   boxes_out (top,8,3) fp32, scores_out (top) fp32 in pick (score) order, count_out: device int = number of boxes written.
 *     Order: descending score, ties by ascending candidate slot, slot = cav * H*W*A + (h*W + w)*A + a (the `top` cut takes the
 *     first `top` in this order).  The reference's argsort()[::-1] leaves ties in an unspecified order.
 *   The filters drop a box with any NaN corner, as the reference's NaN lengths do.  Direction logits: the first largest bin
 *   wins and a NaN never replaces the running best (a NaN in bin 0 keeps bin 0, where torch.max would pick the NaN).
 *   stats_out: device int[2] = anchors above the score threshold, after the size / z filters (NULL allowed)
 *   workspace >= heal_postprocess_workspace(H, W, A, top) bytes; top <= 1320 (the reference uses 1000) */
size_t heal_postprocess_workspace(int H, int W, int anchors_per_cell, int top);
int heal_box_decode_nms(const heal_act_t* cls, const heal_act_t* reg, const heal_act_t* dir, const float* anchors,
                        int H, int W, int anchors_per_cell, float score_threshold, float dir_offset, int num_bins,
                        const float* transform4x4_host, int order_hwl, float nms_threshold, int top,
                        const float* range6_host, float* boxes_out, float* scores_out, int* count_out, int* stats_out,
                        void* workspace, size_t workspace_bytes, void* stream);

/* Late fusion / IoU-aware variant (voxel_postprocessor.py:269-376 with several cavs and `iou_preds`): every cav's heads are decoded
 * with ITS transform (cav -> ego) and anchors, the candidates are concatenated in cav order, then ONE filter + sort + rotated NMS
 * + range mask.  `iou` (optional, (1,H,W,A) logits): score *= ((sigmoid(iou) + 1) / 2)^4 after the threshold test (:343-347); a NaN
 * IoU logit counts as sigmoid 0 (score * 1/16), where the reference's clamp would give a NaN score.  Order and ties as above.
 * cavs_host: HOST array of n_cav descriptors (all maps H x W x anchors_per_cell); workspace >=
 * heal_postprocess_workspace(H * n_cav, W, anchors_per_cell, top). */
typedef struct {
    const heal_act_t* cls; const heal_act_t* reg; const heal_act_t* dir; const heal_act_t* iou;   /* dir / iou may be NULL */
    const float* anchors;                 /* device (H,W,A,7) */
    const float* transform4x4_host;       /* host, row-major 4x4 */
} heal_cav_heads_t;
int heal_box_decode_nms_multi(const heal_cav_heads_t* cavs_host, int n_cav, int H, int W, int anchors_per_cell,
                              float score_threshold, float dir_offset, int num_bins, int order_hwl, float nms_threshold,
                              int top, const float* range6_host, float* boxes_out, float* scores_out, int* count_out,
                              int* stats_out, void* workspace, size_t workspace_bytes, void* stream);

/* Late fusion of one scene as a single capturable call: the same decode, filter, sort, rotated NMS and range mask as
 * heal_box_decode_nms_multi with the cavs in batch order, for cavs that share one anchor grid.  The heads are ONE batched
 * fp32 channels-last map each: cls (n_cav,H,W,A), reg (n_cav,H,W,7A), dir (n_cav,H,W,A*num_bins) or NULL (channel views with
 * cstride / coffset, e.g. the three slices of one fused head output).  transforms_dev: DEVICE fp32 (n_cav,4,4) row-major
 * cav -> ego matrices, read by the decode kernel, so a captured graph picks up new poses.  One decode launch covers every cav.
 * n_cav <= 16; workspace >= heal_postprocess_workspace(H * n_cav, W, anchors_per_cell, top); boxes, scores, count and stats as
 * heal_box_decode_nms.  For the same inputs the boxes, their order and the scores equal heal_box_decode_nms_multi's bit for bit. */
int heal_box_decode_nms_late(const heal_act_t* cls, const heal_act_t* reg, const heal_act_t* dir, const float* anchors,
                             const float* transforms_dev, int n_cav, int H, int W, int anchors_per_cell,
                             float score_threshold, float dir_offset, int num_bins, int order_hwl, float nms_threshold,
                             int top, const float* range6_host, float* boxes_out, float* scores_out, int* count_out,
                             int* stats_out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- detection evaluation: true / false positives of one frame ------------------------------------------------------
 * replaces eval_utils.caluclate_tp_fp (opencood/utils/eval_utils.py:40-92), which opencood/tools/inference.py:171-185 (and
 * inference_w_noise.py, inference_heter_in_order.py) calls once per frame for each of IoU 0.3, 0.5 and 0.7; one call here does up
 * to 8 thresholds.
 *   det_corners (K,8,3) fp32, det_scores (K) fp32, gt_corners (G,8,3) fp32: device.  Only corners 0..3, x and y, are used: the
 *     shapely Polygon of convert_format (common_utils.py:255-270), in fp64 and made counter-clockwise.
 *   thresholds_host: n_thr fp32 IoU thresholds, each > 0.
 *   sorted_scores_out (K) fp32: the scores in descending order.  Ties go by ascending input index (a stable sort) and NaN scores
 *     last.  The reference's np.argsort(-det_score) leaves the order of tied scores unspecified (NumPy's default sort is not
 *     stable and its SIMD dispatch depends on the CPU); this is the one place where the result can differ from the reference's.
 *   tp_out (n_thr, K) uint8: 1 = TP, 0 = FP, per threshold and sorted detection.
 *   status_out: device int, HEAL_EVAL_ZERO_UNION set when a det and a GT have a union of area 0 (two degenerate boxes), where the
 *     reference's compute_iou raises ZeroDivisionError; the flags are then meaningless.
 * Rules, as the reference with NumPy 2: IoU = inter / (area_det + area_gt - inter) in fp64, the det clipped against the GT's
 * edges, rounded once to fp32 (compute_iou, common_utils.py:250-252); boxes whose bounding boxes do not touch have IoU 0.  Dets
 * are taken in score order; a det is FP when no GT is left or when the largest fp32 IoU over the GTs left is below the threshold
 * compared in fp32 (NEP 50 casts the Python float to the array's float32, so an IoU equal to float32(0.7) < 0.7 is a TP; NumPy 1
 * compared in float64), else TP and it takes the GT of that IoU, the lowest GT index on equal IoUs (np.argmax + list.pop).
 * K <= 4096, G <= 4096, 1 <= n_thr <= 8, else HEAL_ERR_ARG.  K = 0 launches nothing (status_out is cleared); G = 0 makes every
 * det FP.  workspace >= heal_eval_workspace(K, G) bytes. */
#define HEAL_EVAL_ZERO_UNION 1
size_t heal_eval_workspace(int K, int G);
int heal_eval_tp_fp(const float* det_corners, const float* det_scores, int K, const float* gt_corners, int G,
                    const float* thresholds_host, int n_thr, float* sorted_scores_out, unsigned char* tp_out, int* status_out,
                    void* ws, size_t ws_bytes, void* stream);

/* The same evaluation with the counts on the device, so that it can follow heal_box_decode_nms in one captured graph (no host
 * read of the box count).  det_count, gt_count: device ints, the live K and G (e.g. the count_out of heal_box_decode_nms).
 * K_cap, G_cap in [1, 4096]: host capacities.  det_corners (K_cap,8,3), det_scores (K_cap), gt_corners (G_cap,8,3): only the
 * leading K / G rows are read.  Outputs at capacity: sorted_scores_out (K_cap), tp_out (n_thr, K_cap) (threshold t at
 * tp_out + t * K_cap), leading K entries written, the rest left as they were.  Rules, tie order, NaN order and
 * HEAL_EVAL_ZERO_UNION as heal_eval_tp_fp: for K <= K_cap and G <= G_cap the leading K scores and flags of every threshold equal
 * heal_eval_tp_fp's on the leading rows bit for bit.  A count below 0 or above its capacity sets HEAL_EVAL_OVER_CAPACITY and
 * writes no score and no flag (the counts are never clamped).  workspace >= heal_eval_workspace(K_cap, G_cap) bytes.  Launches
 * four kernels whatever the counts; every argument is checked on the host (HEAL_ERR_ARG), nothing is read back. */
#define HEAL_EVAL_OVER_CAPACITY 2
int heal_eval_tp_fp_counted(const float* det_corners, const float* det_scores, const int* det_count, int K_cap,
                            const float* gt_corners, const int* gt_count, int G_cap, const float* thresholds_host, int n_thr,
                            float* sorted_scores_out, unsigned char* tp_out, int* status_out, void* ws, size_t ws_bytes,
                            void* stream);

/* ---- format conversion between fp32 and (split-)bf16 channels-last buffers -------------------
 * Any views: 4 channels at a time when channels, both channel strides and offsets (and split plane strides) are multiples of 4
 * and both data pointers are 16-byte aligned (fp32) or 8-byte aligned (bf16 / split), one channel at a time otherwise (same
 * results).  fp32 -> bf16 rounds to nearest even; fp32 -> split is hi = bf16(x), lo = bf16(x - hi); split -> fp32 is hi + lo.
 * num_pixels = 0 launches nothing (the data pointers may be NULL). */
int heal_act_convert(const heal_act_t* src, const heal_act_t* dst, size_t num_pixels, int channels, void* stream);

/* ---- agent assembly of a heterogeneous scene ------------------------------------------------------
 * replaces the per-agent convert + camera CenterCrop + torch.cat of HeterPyramidCollab / HeterModelBaseline /
 * HeterModelBaselineMs.forward (heter_pyramid_collab.py:147-161, heter_model_baseline.py:117-130,
 * heter_model_baseline_ms.py:110-123): agent a of the (num_agents, H, W, channels) `dst` is image agent_image_host[a] of source
 * agent_source_host[a].  One source per modality: its (images, height, width, channels) map in any format.  A source with
 * center_crop = 0 must be H x W and is copied; with center_crop = 1 it is cut to H x W as torchvision CenterCrop does: per axis
 * of source size s and target t, zero padding of (t - s) // 2 before and (t - s + 1) // 2 after when t > s, else a window at
 * int(round((s - t) / 2.0)) (Python rounding, halves to even).  Values are converted exactly as heal_act_convert converts
 * them (dst in any format; padding is +0).  Sources, positions and sizes are host metadata copied into the launch, so the call
 * can be captured.  4 channels at a time when channels and every view meet heal_act_convert's vector rule, one channel at a
 * time otherwise (same results).  1 <= num_sources <= 8 and 1 <= num_agents <= 64 (HEAL_ERR_UNSUPPORTED above); a NULL data
 * pointer, a format outside 0..2, cstride < coffset + channels, an agent index out of range or a center_crop = 0 source of
 * another size is HEAL_ERR_ARG. */
#define HEAL_AGENT_STACK_MAX_SOURCES 8
#define HEAL_AGENT_STACK_MAX_AGENTS 64
typedef struct {
    heal_act_t map;
    int images, height, width;
    int center_crop;
} heal_stack_source_t;
int heal_agent_stack(const heal_stack_source_t* sources_host, int num_sources, const int* agent_source_host,
                     const int* agent_image_host, int num_agents, int channels, const heal_act_t* dst, int H, int W,
                     void* stream);

/* ---- ConvNeXt aligner (SURVEY.md 8f-3) -------------------------------------------------------------
 * depthwise k x k conv (+bias) + LayerNorm over channels, one kernel: the front half of ConvNeXtBlock.forward
 * (opencood/models/sub_modules/feature_alignnet_modules.py:331-336, LayerNorm :12-25 channels_last, biased variance).
 *   dw_weight [k*k][C] fp32 (tap-major, read as float2: 8-byte aligned, else HEAL_ERR_UNSUPPORTED), dw_bias [C] or NULL,
 *   ln_weight / ln_bias [C]; C in {64,128,192,256}
 * The two Linear layers that follow are 1x1 convolutions on heal_conv2d_tc (`relu` = 2 selects the exact erf GELU in the
 * epilogue; layer scale `gamma` folded into the second one; the block's residual add is the conv's residual input). */
int heal_dwconv_layernorm(const heal_act_t* in, int N, int H, int W, int C, const float* dw_weight, const float* dw_bias,
                          int ksize, const float* ln_weight, const float* ln_bias, float eps, const heal_act_t* out, void* stream);

/* 3x3 / stride 2 / pad 1 max pooling, channels-last (torchvision ResNet stem of CamEncode_Resnet101,
 * opencood/models/sub_modules/lss_submodule.py:196-199).  depth_to_space_in != 0: the logical (N,H,W,C) input is stored as
 * (N,H/2,W/2,4C) with channel block (y&1)*2+(x&1) -- the phase-major output of the space-to-depth form of the 7x7/2 stem conv.
 * Reads and writes 4 channels at a time: C, channel strides, offsets (and split plane strides) multiples of 4 and in->data /
 * out->data 16-byte aligned (fp32) or 8-byte aligned (bf16 / split), else HEAL_ERR_UNSUPPORTED. */
int heal_maxpool3x3s2(const heal_act_t* in, int N, int H, int W, int C, int depth_to_space_in, const heal_act_t* out, void* stream);

/* ---- EfficientNet-B0 camera trunk of Lift-Splat-Shoot (`camera_encoder: EfficientNet`, SURVEY.md 8c) ---------------------
 * opencood/models/sub_modules/lss_submodule.py:87-111 runs efficientnet_pytorch's stem and MBConv blocks, then `Up` (:17-36).
 * Trunk tensors are dense channels-last fp32 (N,H,W,C); BatchNorm (eps 1e-3) is folded into weight / bias by the caller;
 * swish(x) = x * sigmoid(x).  Channel counts are multiples of 4.
 *
 * heal_stem_conv_swish: 3x3 / stride 2 conv 3 -> 32 reading the first 3 of `image_channels` planes of the NCHW image, zero pad
 *   0 before and 1 after in y and x (the package's static "same" padding), + bias, swish.  weight [27][32], row (ci*3+ky)*3+kx.
 *   out (N, (H-2)/2+1, (W-2)/2+1, 32).
 * heal_dwconv_bn_swish: depthwise ksize in {3,5}, stride in {1,2}, `pad_top` / `pad_left` zeros before the image (what lies after
 *   follows from Ho, Wo), + bias, swish.  weight [ksize*ksize][C] tap-major.  Also writes sums (N,C) = the sum of `out` over its
 *   pixels, added in a fixed order (bit-identical run to run).  workspace >= heal_dwconv_bn_swish_workspace(N, C, Ho, Wo).
 * heal_se_gate: gate (N,C) = sigmoid(W_e swish(W_r (sums / HW) + b_r) + b_e).  w_reduce [Csq][C], w_expand_t [Csq][C]
 *   (the expand weight transposed); C <= 1152, Csq <= 64.
 * heal_pwconv: 1x1 conv out = act(sum_ci in[.., ci] * gate[n, ci] * weight[ci][co] + bias[co]) + residual.  weight [Cin][Cout];
 *   gate (N,Cin) or NULL; swish_epilogue 0 | 1; residual (N,HW,Cout) or NULL.
 * heal_upsample2x_concat: out (N, 2*H1, 2*W1, Cout) = [x2 (C2 channels) | bilinear x2, align_corners=True, of x1 (C1 channels) |
 *   zeros]; any storage format on each side (the zero tail pads the channel count for the tensor-core convolution that follows). */
int heal_stem_conv_swish(const float* image, int N, int image_channels, int H, int W, const float* weight, const float* bias,
                         float* out, void* stream);
size_t heal_dwconv_bn_swish_workspace(int N, int C, int Ho, int Wo);
int heal_dwconv_bn_swish(const float* in, int N, int H, int W, int C, const float* weight, const float* bias, int ksize,
                         int stride, int pad_top, int pad_left, int Ho, int Wo, float* out, float* sums,
                         void* workspace, size_t workspace_bytes, void* stream);
int heal_se_gate(const float* sums, int N, int C, int Csq, int HW, const float* w_reduce, const float* b_reduce,
                 const float* w_expand_t, const float* b_expand, float* gate, void* stream);
int heal_pwconv(const float* in, int N, int HW, int Cin, int Cout, const float* weight, const float* bias, const float* gate,
                int swish_epilogue, const float* residual, float* out, void* stream);
int heal_upsample2x_concat(const heal_act_t* x1, const heal_act_t* x2, int N, int H1, int W1, int C1, int C2,
                           const heal_act_t* out, int Cout, void* stream);

/* ---- peer-to-peer exchange over NVLink / NVSwitch (agent-per-GPU partition, SURVEY.md 8e) ---------------------
 * The buffers are SYMMETRIC: every rank allocated the same size and mapped every peer's copy (peer_*_host[r] = this process's
 * device pointer to rank r's copy; [self] = the local one).
 * heal_p2p_push: copy `bytes` (multiple of 16) from src_local to peer_dst_host[r] for every r != self (same offset everywhere).
 * heal_p2p_signal_wait: ++seq_dev[0]; store it (release, system scope) into flags[self] of every rank's flag array
 *   (world u32 each); wait until the local flag array holds >= that value for every rank.  One thread block; capturable. */
int heal_p2p_push(const void* src_local, void* const* peer_dst_host, int world, int self, size_t bytes, void* stream);
int heal_p2p_signal_wait(void* const* peer_flags_host, int world, int self, unsigned* seq_dev, void* stream);

/* ---- on-GPU input path (SURVEY.md 8f-4): the reference's host-side point filters before voxelisation ----------------
 * shuffle_points / mask_ego_points / mask_points_by_range (opencood/utils/pcd_utils.py:41-95, applied in this order by
 * intermediate_heter_fusion_dataset.py:141-173) as one stable compaction per agent: points_out = mask(points[perm]).
 *   points (P,4) f32, agents concatenated; perm (P) i32 GLOBAL source index per slot (the host-drawn shuffle) or NULL;
 *   agent_offsets (A+1) i32 device (live count = offsets[A] <= P; rows before offsets[0] are dropped, so
 *   agent_offsets_out[0] = 0); range6_host = [xmin,ymin,zmin,xmax,ymax,zmax] (strict);
 *   remove_ego != 0 drops the ego-vehicle box.  points_out (P,4); agent_offsets_out (A+1) i32 device. */
size_t heal_mask_points_workspace(int num_points);
int heal_mask_points(const float* points, const int* perm, const int* agent_offsets, int num_agents, int num_points,
                     const float* range6_host, int remove_ego, float* points_out, int* agent_offsets_out,
                     void* workspace, size_t workspace_bytes, void* stream);

/* The camera agent's image stage (SURVEY.md 8f-4): the reference's inference resize, crop and normalisation, done per camera on
 * the host in its DataLoader workers (intermediate_heter_fusion_dataset.py:199-246; camera_utils.py:33-59 sample_augmentation
 * with is_train False, :62-91 img_transform = PIL resize with its default antialiased bicubic filter, then crop; :120-125
 * normalize_img = ToTensor + Normalize(ImageNet mean / std)).  Bit-exact: Pillow's 8-bit fixed-point resample (horizontal pass,
 * clipped to uint8, then vertical pass), black outside the resized frame, then (u / 255 - mean) / std in fp32.
 *   frames      (n_img, H0, W0, 3) uint8, HWC as decoded; every camera of every agent of one modality in one call
 *   col_table   (fW, 2 + col_taps) i32: per output column, the first source column, the tap count and col_taps int32 taps
 *               (1 << 22 = 1.0); entry i is column crop_left + i of the resized frame, so the crop box is folded into the table
 *               and a count of 0 marks a column outside the resized frame.  An axis that keeps its size has one tap of 1 << 22.
 *   row_table   (fH, 2 + row_taps) i32: the same per output row
 *   span_rows   the most source rows one 32-row band of output rows needs (sizes the shared tile; the host computes it)
 *   layout 0    out (n_img, 3, fH, fW) fp32 NCHW (heal_stem_conv_swish reads it)
 *   layout 1    out (n_img, fH/4, fW/4, 64) fp32 channels-last, channel c*16 + dy*4 + dx, c == 3 zero: the space-to-depth input of
 *               the ResNet-101 stem (fH, fW multiples of 8)
 * No atomics, no host sync: the same bits on every run. */
int heal_camera_input(const uint8_t* frames, int n_img, int H0, int W0, const int* col_table, int col_taps,
                      const int* row_table, int row_taps, int fH, int fW, int span_rows, int layout, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HEAL_B200_H_ */
