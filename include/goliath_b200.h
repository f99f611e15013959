/*
 * include/goliath_b200.h — C ABI of libgoliath_b200.so (hand-written sm_90a kernels).
 *
 * The drop-in boundary of the goliath render hot path (SURVEY.md §8b).  Every entry point
 *   - takes raw DEVICE pointers (fp32 / int32 / int64, contiguous, layouts exactly as the reference's
 *     tensors), plain sizes and a cudaStream_t passed as void*;
 *   - runs on the CURRENT device of the calling thread and only on the given stream (the reference's
 *     mvpraymarchlib/utilslib launch on stream 0 with no device guard, mvpraymarch.cpp:122,142,176 —
 *     this ABI is the superset behaviour needed for one-process-per-GPU operation);
 *   - never allocates or synchronises: the caller owns outputs, gradients and workspaces;
 *   - returns 0, or the cudaError_t value of the failing launch / argument check.
 * Each declaration names the reference binding it replaces.  The Python-side bindings that mirror the
 * reference's pybind modules live in goliath_b200/{sgutilslib,mvpraymarchlib,utilslib}.py and
 * goliath_b200/gsplat/; INTEGRATION.md shows the stub a goliath maintainer would add.
 */
#ifndef GOLIATH_B200_H_
#define GOLIATH_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* library/ABI version: major*1000 + minor */
int gb_version(void);
/* kernels launched by this library since load / last reset (host counter; bench.py gpu_launches) */
unsigned long long gb_launch_count(void);
void gb_launch_count_reset(void);

/* ---------------------------------------------------------------- sgutilslib (extensions/sgutils/sg.cu) */

/* replaces sgutilslib.evaluate_gaussian_fwd — sg.cu:177-224 (kernel :27-76).
 * lobe_dirs [N,D,3] (already normalised by sgutils.py:75), lobe_sigmas [N,D], light_values [N,L,3],
 * light_pts [N,L,3], prim_pts [N,D,3], n_lights [N] int32, integral [N,D,3] out. w_type in 0..3. */
int gb_sg_evaluate_fwd(const float* lobe_dirs, const float* lobe_sigmas, const float* light_values,
                       const float* light_pts, const float* prim_pts, const int32_t* n_lights, float* integral,
                       int N, int D, int L, int w_type, void* stream);

/* replaces sgutilslib.evaluate_gaussian_bwd — sg.cu:226-277 (kernel :78-175).
 * grad_dirs [N,D,3], grad_sigmas [N,D] are overwritten; grad_light_values [N,L,3] may be NULL, otherwise it
 * is accumulated into (the reference zero-fills it in sgutils.py:43-47). */
int gb_sg_evaluate_bwd(const float* lobe_dirs, const float* lobe_sigmas, const float* light_values,
                       const float* light_pts, const float* prim_pts, const int32_t* n_lights,
                       const float* grad_integral, float* grad_dirs, float* grad_sigmas, float* grad_light_values,
                       int N, int D, int L, int w_type, void* stream);

/* ---------------------------------------------------------------- gsplat 0.1.11 (third-party; call sites
 * ca_code/utils/render_gsplat.py:49-63, 65-78, 90-104) */

/* replaces gsplat._C.project_gaussians_forward.  means3d [G,3], scales [G,3], quats [G,4] (w,x,y,z),
 * viewmat: DEVICE pointer to >= 12 floats, row-major [R|t].  Outputs (all written for every Gaussian;
 * culled ones get zeros): cov3d [G,6], xys [G,2], depths [G], radii [G] i32, conics [G,3],
 * compensation [G], num_tiles_hit [G] i32. */
int gb_project_gaussians_fwd(int G, const float* means3d, const float* scales, float glob_scale,
                             const float* quats, const float* viewmat, float fx, float fy, float cx, float cy,
                             int img_h, int img_w, int block_width, float clip_thresh, float* cov3d, float* xys,
                             float* depths, int32_t* radii, float* conics, float* compensation,
                             int32_t* num_tiles_hit, void* stream);

/* gb_project_gaussians_fwd that also zeroes grad_acc [10 G] fp32, the fused render's blend-backward accumulator:
 * v_rgbd [G,4] | v_xy [G,2] | v_conic [G,3] | v_opacity_eff [G]. */
int gb_project_gaussians_fwd_acc(int G, const float* means3d, const float* scales, float glob_scale,
                                 const float* quats, const float* viewmat, float fx, float fy, float cx, float cy,
                                 int img_h, int img_w, int block_width, float clip_thresh, float* cov3d, float* xys,
                                 float* depths, int32_t* radii, float* conics, float* compensation,
                                 int32_t* num_tiles_hit, float* grad_acc, void* stream);

/* The fused render's per-Gaussian backward in one pass: grad_acc (gb_project_gaussians_fwd_acc's layout, filled by the
 * blend backward), opacity [G] and the projection's saved tensors -> v_colors [G,3], v_opacity [G], v_mean3d,
 * v_scale, v_quat; the same bits as gb_splat_grad_unpack followed by gb_project_gaussians_bwd. */
int gb_splat_project_bwd(int G, const float* means3d, const float* scales, float glob_scale, const float* quats,
                         const float* viewmat, float fx, float fy, const float* cov3d, const int32_t* radii,
                         const float* conics, const float* compensation, const float* opacity, const float* grad_acc,
                         float* v_colors, float* v_opacity, float* v_mean3d, float* v_scale, float* v_quat,
                         void* stream);

/* replaces gsplat._C.project_gaussians_backward.  All five gradient outputs are overwritten. */
int gb_project_gaussians_bwd(int G, const float* means3d, const float* scales, float glob_scale,
                             const float* quats, const float* viewmat, float fx, float fy, const float* cov3d,
                             const int32_t* radii, const float* conics, const float* compensation,
                             const float* v_xy, const float* v_depth, const float* v_conic,
                             const float* v_compensation, float* v_cov2d, float* v_cov3d, float* v_mean3d,
                             float* v_scale, float* v_quat, void* stream);

/* replaces gsplat.utils.compute_cumulative_intersects (torch.cumsum int32): inclusive scan. */
size_t gb_cumsum_workspace_bytes(int n);
int gb_cumsum_i32(int n, const int32_t* in, int32_t* out, void* workspace, void* stream);

/* replaces gsplat._C.map_gaussian_to_intersects: isect_ids [I] int64 = (tile_id << 32) | bits(depth),
 * gaussian_ids [I] int32, emitted per Gaussian in row-major tile order. */
int gb_map_gaussian_to_intersects(int G, const float* xys, const float* depths, const int32_t* radii,
                                  const int32_t* cum_tiles_hit, int img_h, int img_w, int block_width,
                                  int64_t* isect_ids, int32_t* gaussian_ids, void* stream);

/* replaces torch.sort(isect_ids) + gather in gsplat.utils.bin_and_sort_gaussians: stable ascending radix
 * sort on the low key_bits bits (32 + ceil(log2(#tiles))). */
size_t gb_sort_workspace_bytes(int64_t n);
int gb_sort_intersects(int64_t n, const int64_t* isect_ids, const int32_t* gaussian_ids, int64_t* isect_sorted,
                       int32_t* gids_sorted, int key_bits, void* workspace, void* stream);

/* replaces gsplat._C.get_tile_bin_edges: tile_bins [T,2] int32, zeroed by the caller. */
int gb_get_tile_bin_edges(int64_t n, const int64_t* isect_sorted, int32_t* tile_bins, void* stream);

/* replaces gsplat._C.rasterize_forward (channels == 3); channels == 4 is the fused rgb+depth pass.
 * colors [G,C], opacities [G], background [C] (device).  out_img [H,W,C], final_Ts [H,W],
 * final_idx [H,W] i32 are fully overwritten. */
int gb_rasterize_fwd(int img_h, int img_w, int block_width, int channels, const int32_t* gids_sorted,
                     const int32_t* tile_bins, const float* xys, const float* conics, const float* colors,
                     const float* opacities, const float* background, float* out_img, float* final_Ts,
                     int32_t* final_idx, void* stream);

/* replaces gsplat._C.rasterize_backward.  v_xy [G,2], v_conic [G,3], v_colors [G,C], v_opacity [G] are
 * accumulated into (caller zeroes them).  v_output_alpha [H,W] may be NULL (no gradient through alpha) here and in every
 * gb_rasterize_*_bwd below. */
int gb_rasterize_bwd(int img_h, int img_w, int block_width, int channels, const int32_t* gids_sorted,
                     const int32_t* tile_bins, const float* xys, const float* conics, const float* colors,
                     const float* opacities, const float* background, const float* final_Ts,
                     const int32_t* final_idx, const float* v_output, const float* v_output_alpha, float* v_xy,
                     float* v_conic, float* v_colors, float* v_opacity, void* stream);

/* ---- packed blend path (block_width == 16): same results as gb_rasterize_fwd/bwd, different work distribution.
 * These have no counterpart in gsplat's binding; they sit behind the same rasterize_gaussians call
 * (ca_code/utils/render_gsplat.py:65-78,90-104). */

/* gather (xy, conic, opacity, colours, cull box) of every intersection in sorted order: records [n,12] fp32 */
int gb_pack_records(int64_t n, int channels, const int32_t* gids_sorted, const float* xys, const float* conics,
                    const float* colors, const float* opacities, float* records, void* stream);

/* fused-render variant: record opacity = opacity*compensation (render_gsplat.py:72), 4th colour = depth (:97) */
int gb_pack_records_fused(int64_t n, const int32_t* gids_sorted, const float* xys, const float* conics,
                          const float* colors3, const float* depths, const float* opacity, const float* compensation,
                          float* records, void* stream);

/* multi-condition (OLAT) renders: the lighting conditions of a view share geometry, projection and tile lists
 * (ca_code/utils/light_decorator.py:167 feeds the same avatar under one light at a time); this rewrites only the colour
 * quarter of the fused-render records in place: records[i].c = (colors3[gids_sorted[i]], depths[gids_sorted[i]]).
 * n_dev: device int32 count of valid records (may be NULL: cap records). */
int gb_records_set_colors(int64_t cap, const int32_t* n_dev, const int32_t* gids_sorted, const float* colors3,
                          const float* depths, float* records, void* stream);

/* four lighting conditions per blend pass (OLAT, BASELINE config 3): the conditions of a view share every alpha and
 * transmittance, so one walk of the tile lists blends four colour sets (csrc/splat_blend_mom.cu).  "Wide" records [cap,20]
 * fp32 = the 32-byte geometry of the packed records + 4 x rgb; gb_records_widen copies the geometry once per view,
 * gb_records_set_colors4 rewrites the colour part per group of (up to 4) conditions from nk consecutive [G,3] tables. */
int gb_records_widen(int64_t cap, const int32_t* n_dev, const float* records, float* records_wide, void* stream);
int gb_records_set_colors4(int64_t cap, const int32_t* n_dev, const int32_t* gids_sorted, const float* colors, int nk,
                           int64_t G, float* records_wide, void* stream);
/* out_planes [4][H][W][3] (3-channel background added to each). */
int gb_rasterize_multi_fwd(int img_h, int img_w, const int32_t* tile_bins, const int32_t* tile_order, int sched,
                           const float* records_wide, const float* background, float* out_planes, void* stream);
/* v_planes [4][H][W][3]; final_Ts / final_idx from the view's single-condition pass; v_xy / v_conic / v_opacity accumulated;
 * v_colors12 [G,12] (zero-filled): the four colour gradients interleaved per Gaussian, split by gb_colors12_unpack (which
 * also clears it for the next group). */
int gb_rasterize_multi_bwd(int img_h, int img_w, const int32_t* gids_sorted, const int32_t* tile_bins,
                           const int32_t* tile_order, int sched, const float* records_wide, const float* background,
                           const float* final_Ts, const int32_t* final_idx, const float* v_planes, float* v_xy, float* v_conic,
                           float* v_colors12, float* v_opacity, void* stream);
int gb_colors12_unpack(int64_t G, int nk, float* v_colors12, float* v_colors, void* stream);

/* backward glue of the fused render: split v_colors4 / v_opacity_eff into v_colors3, v_opacity, v_comp, v_depth */
int gb_splat_grad_unpack(int G, const float* v_colors4, const float* v_opac_eff, const float* opacity,
                         const float* compensation, float* v_colors3, float* v_opacity, float* v_comp, float* v_depth,
                         void* stream);

/* ---- sync-free ("_dn": device-side n) variants: the intersection count stays on the device (n_dev = last element of
 * cum_tiles_hit), buffers hold `cap` intersections, *overflow is set when the true count exceeds cap.  They remove
 * the host synchronisation the reference performs (gsplat utils: cum_tiles_hit[-1].item()) and make the whole render
 * capturable in a CUDA graph. */
int gb_map_gaussian_to_intersects_dn(int G, const float* xys, const float* depths, const int32_t* radii,
                                     const int32_t* cum_tiles_hit, int img_h, int img_w, int block_width, int64_t cap,
                                     int64_t* isect_ids, int32_t* gaussian_ids, void* stream);
int gb_sort_intersects_dn(int64_t cap, const int32_t* n_dev, const int64_t* isect_ids, const int32_t* gaussian_ids,
                          int64_t* isect_sorted, int32_t* gids_sorted, int key_bits, void* workspace, void* stream);
int gb_get_tile_bin_edges_dn(int64_t cap, const int32_t* n_dev, const int64_t* isect_sorted, int32_t* tile_bins,
                             int32_t* overflow, void* stream);
int gb_pack_records_fused_dn(int64_t cap, const int32_t* n_dev, const int32_t* gids_sorted, const float* xys,
                             const float* conics, const float* colors3, const float* depths, const float* opacity,
                             const float* compensation, float* records, void* stream);

/* gb_bin_tiles_pack has one formulation (per-tile buckets, each sorted by (depth, id) in shared memory): both getters
 * return 0 and both setters accept and ignore any value.  Kept so that callers which label or select modes work. */
int gb_get_rank_sort_mode(void);
int gb_get_tile_sort_mode(void);
void gb_set_tile_sort_mode(int mode);
void gb_set_rank_sort_mode(int mode);

/* Bucket binning of the fused render (csrc/splat_bin_tiles.cu): replaces, for the fused path, the whole of gsplat
 * 0.1.11 bin_and_sort_gaussians (compute_cumulative_intersects, map_gaussian_to_intersects, torch.sort,
 * get_tile_bin_edges — call sites ca_code/utils/render_gsplat.py:65-78,90-104) plus the record packing, with the same
 * bit-exact outputs: intersections are bucketed per tile with atomics (Gaussian ids), and one CTA per tile sorts its
 * bucket by (depth key, id) with a radix sort in shared memory (tiles longer than 5120 entries: through global memory).  Outputs: tile_bins [T,2], tile_order [T]
 * (tile_sched = 1: an SM-affine schedule of gb_tile_schedule_ints(T) int32 instead, see gb_tile_schedule),
 * gids_sorted [cap], records [cap,12]; n_out (device int32, may be NULL) = true intersection count; *overflow = 1
 * when it exceeds cap (the excess is dropped).  Sync-free, never allocates, capturable in a CUDA graph. */
int gb_bin_tiles_supported(int G); /* 1 for 1 <= G <= 1.5 x 2^20 (1572864) Gaussians per view */
size_t gb_bin_tiles_workspace_bytes(int G, int num_tiles, int64_t cap);
int gb_bin_tiles_pack(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                      const float* colors3, const float* opacity, const float* compensation, int img_h, int img_w,
                      int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order, int tile_sched,
                      int32_t* gids_sorted, float* records, int32_t* n_out, int32_t* overflow, void* workspace,
                      void* stream);
/* Same, with colors3 allowed to arrive late: colors_ready (cudaEvent_t recorded on the stream that writes colors3, or
 * NULL) is waited for on `stream` just before the first kernel that reads colors3 (a small kernel after the per-tile
 * sort), so counts, buckets and the per-tile sort run beside the caller's shade (rgca.py:557-575 precedes
 * render_gsplat.py:65 in the reference; only the colours depend on it). */
int gb_bin_tiles_pack_ev(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                         const float* colors3, const float* opacity, const float* compensation, int img_h, int img_w,
                         int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order, int tile_sched,
                         int32_t* gids_sorted, float* records, int32_t* n_out, int32_t* overflow, void* workspace,
                         void* colors_ready, void* stream);

/* Binning WITHOUT the sorted-record gather, for gb_rasterize_ranked_fwd/bwd: ranks_sorted [cap] (per tile, the Gaussian
 * ids in blend order), rec_by_rank [G,12] (one 48-byte record per visible Gaussian, at its id) and rank_to_gid [G] (the
 * identity: ranks_sorted already holds ids) are written to the CALLER's arrays (they must live until the backward).  Everything else as gb_bin_tiles_pack_ev.  No
 * counterpart in gsplat: it replaces the per-intersection sorted arrays of bin_and_sort_gaussians by per-Gaussian ones. */
int gb_bin_tiles_ranked(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                        const float* colors3, const float* opacity, const float* compensation, int img_h, int img_w,
                        int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order, int tile_sched,
                        int32_t* ranks_sorted, float* rec_by_rank, int32_t* rank_to_gid, int32_t* n_out, int32_t* overflow,
                        void* workspace, void* colors_ready, void* stream);
/* Blend straight from the by-id table of gb_bin_tiles_ranked (csrc/splat_blend_mom.cu, RANKED staging: 16-byte cp.async
 * gathers by list entry into the stage ring instead of bulk copies of materialised sorted records).  Same results as
 * gb_rasterize_packed_fwd/bwd; final_idx indexes ranks_sorted.  The backward takes each hit's Gaussian id from
 * ranks_sorted and does not read rank_to_gid (kept in the signature; gb_bin_tiles_ranked writes it as the identity).  channels 3 or 4; tile_order = launch order (gb_tile_order) or NULL. */
int gb_rasterize_ranked_fwd(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order,
                            const int32_t* ranks_sorted, const float* rec_by_rank, const float* background,
                            float* out_img, float* final_Ts, int32_t* final_idx, void* stream);
int gb_rasterize_ranked_bwd(int img_h, int img_w, int channels, const int32_t* rank_to_gid, const int32_t* ranks_sorted,
                            const int32_t* tile_bins, const int32_t* tile_order, const float* rec_by_rank,
                            const float* background, const float* final_Ts, const int32_t* final_idx,
                            const float* v_output, const float* v_output_alpha, float* v_xy, float* v_conic,
                            float* v_colors, float* v_opacity, void* stream);
/* The ranked pair with a backward that does not cull the tiles again: gb_rasterize_ranked_fwd_lists is
 * gb_rasterize_ranked_fwd (identical out_img / final_Ts / final_idx) that also stores each pixel warp's footprint hits,
 * as sorted indices into ranks_sorted, in hit_list [8 cap] int32 (warp w of a tile with range [x, y) at 8x + w(y - x))
 * and in hit_count [16 T + 2] int32 the number of them the backward needs (hit_count[0 .. 8 T)); the rest of
 * hit_count is the backward's work space (a draw counter the forward zeroes, and the (tile, warp) items ordered by hit
 * count).  gb_rasterize_ranked_bwd_lists walks those lists back to front, one work item per (tile, pixel warp),
 * heaviest items first, and gives gb_rasterize_ranked_bwd's gradients up to the order of the atomic adds; it may be run
 * again on the same lists. */
int gb_rasterize_ranked_fwd_lists(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order,
                                  const int32_t* ranks_sorted, const float* rec_by_rank, const float* background,
                                  float* out_img, float* final_Ts, int32_t* final_idx, int32_t* hit_list,
                                  int32_t* hit_count, void* stream);
int gb_rasterize_ranked_bwd_lists(int img_h, int img_w, int channels, const int32_t* ranks_sorted,
                                  const int32_t* tile_bins, const int32_t* hit_list,
                                  int32_t* hit_count, const float* rec_by_rank, const float* background,
                                  const float* final_Ts, const int32_t* final_idx, const float* v_output,
                                  const float* v_output_alpha, float* v_xy, float* v_conic, float* v_colors,
                                  float* v_opacity, void* stream);

/* The head step's pair: gb_bin_tiles_buckets is gb_bin_tiles_ranked (launch-order tiles) without the per-tile sort: it
 * leaves each tile's Gaussian ids in arbitrary order in bucket [cap] int32 and their 32-bit depth keys at the same
 * slots of ranks_keys [cap] int32.  gb_rasterize_ranked_fwd_sort_lists sorts each tile's bucket by (depth key, id) in
 * the CTA that then blends it, writes the sorted ids over ranks_keys (then identical to gb_bin_tiles_ranked's
 * ranks_sorted) and gives gb_rasterize_ranked_fwd_lists' out_img, final_Ts, final_idx, hit_list and hit_count.
 * depths [G] are the same depths the binning took.  gb_rasterize_ranked_bwd_lists runs on the result unchanged. */
int gb_bin_tiles_buckets(int G, const float* xys, const float* depths, const int32_t* radii, const float* conics,
                         const float* colors3, const float* opacity, const float* compensation, int img_h, int img_w,
                         int block_width, int64_t cap, int32_t* tile_bins, int32_t* tile_order, int32_t* ranks_keys,
                         int32_t* bucket, float* rec_by_rank, int32_t* rank_to_gid, int32_t* n_out, int32_t* overflow,
                         void* workspace, void* colors_ready, void* stream);
int gb_rasterize_ranked_fwd_sort_lists(int img_h, int img_w, int channels, const int32_t* tile_bins,
                                       const int32_t* tile_order, const float* depths, int32_t* bucket,
                                       int32_t* ranks_keys, const float* rec_by_rank, const float* background,
                                       float* out_img, float* final_Ts, int32_t* final_idx, int32_t* hit_list,
                                       int32_t* hit_count, void* stream);
/* The head view finished inside the blend kernels.  gb_rasterize_ranked_fwd_sort_finish is
 * gb_rasterize_ranked_fwd_sort_lists (4 channels) writing rgb [3,H,W], alpha [H,W] = 1 - final_Ts and depth [H,W] =
 * depth channel / clamp(alpha, 0.05, 1) instead of the 4-channel image: gb_render_finish_fwd's results, bit for bit.
 * gb_rasterize_ranked_bwd_lists_finish is gb_render_finish_bwd + gb_rasterize_ranked_bwd_lists on g_rgb [3,H,W] and
 * g_depth [H,W] (either may be NULL); alpha takes no gradient.  background holds 3 floats in both. */
int gb_rasterize_ranked_fwd_sort_finish(int img_h, int img_w, const int32_t* tile_bins, const int32_t* tile_order,
                                        const float* depths, int32_t* bucket, int32_t* ranks_keys,
                                        const float* rec_by_rank, const float* background, float* rgb, float* alpha,
                                        float* depth, float* final_Ts, int32_t* final_idx, int32_t* hit_list,
                                        int32_t* hit_count, void* stream);
int gb_rasterize_ranked_bwd_lists_finish(int img_h, int img_w, const int32_t* ranks_sorted, const int32_t* tile_bins,
                                         const int32_t* hit_list, int32_t* hit_count, const float* rec_by_rank,
                                         const float* background, const float* final_Ts, const int32_t* final_idx,
                                         const float* alpha, const float* g_rgb, const float* g_depth, float* v_xy,
                                         float* v_conic, float* v_colors, float* v_opacity, void* stream);

/* launch order of the tiles, longest list first: order [T] int32 */
int gb_tile_order(int num_tiles, const int32_t* tile_bins, int32_t* order, void* stream);

/* blend formulation: 0 = CTA-synchronous double buffer (csrc/splat_blend_packed.cu), 1 = warp-decoupled mbarrier
 * pipeline (csrc/splat_blend_pipe.cu), 2 = the pipeline over an SM-affine tile schedule; environment
 * GOLIATH_B200_BLEND=batch|pipe|affine.  gb_rasterize_packed_fwd/bwd launch the CTA-synchronous kernels in mode 0 and
 * the pipeline otherwise; callers that build a schedule use gb_rasterize_sched_fwd/bwd in mode 2.  Outputs are
 * identical in every mode: pixels bit for bit, gradients to atomics order. */
int gb_get_blend_mode(void);
void gb_set_blend_mode(int mode);

/* SM-affine schedule of the tiles (one work queue per SM, near-equal sums of list lengths): sched holds
 * gb_tile_schedule_ints(num_tiles) int32; consumed by gb_rasterize_sched_fwd/bwd, which take the same arguments as
 * gb_rasterize_packed_fwd/bwd and give the same outputs. */
int gb_tile_schedule_ints(int num_tiles);
int gb_tile_schedule(int num_tiles, const int32_t* tile_bins, int32_t* sched, void* stream);
int gb_rasterize_sched_fwd(int img_h, int img_w, int channels, const int32_t* tile_bins, int32_t* sched,
                           const float* records, const float* background, float* out_img, float* final_Ts,
                           int32_t* final_idx, void* stream);
int gb_rasterize_sched_bwd(int img_h, int img_w, int channels, const int32_t* gids_sorted, const int32_t* tile_bins,
                           int32_t* sched, const float* records, const float* background, const float* final_Ts,
                           const int32_t* final_idx, const float* v_output, const float* v_output_alpha, float* v_xy,
                           float* v_conic, float* v_colors, float* v_opacity, void* stream);

/* blend forward over packed records streamed with cp.async.bulk; tile_order may be NULL */
int gb_rasterize_packed_fwd(int img_h, int img_w, int channels, const int32_t* tile_bins, const int32_t* tile_order,
                            const float* records, const float* background, float* out_img, float* final_Ts,
                            int32_t* final_idx, void* stream);

/* blend backward over packed records; gradients are accumulated into (caller zeroes them) */
int gb_rasterize_packed_bwd(int img_h, int img_w, int channels, const int32_t* gids_sorted,
                            const int32_t* tile_bins, const int32_t* tile_order, const float* records,
                            const float* background, const float* final_Ts, const int32_t* final_idx,
                            const float* v_output, const float* v_output_alpha, float* v_xy, float* v_conic,
                            float* v_colors, float* v_opacity, void* stream);

/* ---------------------------------------------------------------- utilslib (extensions/utils) */

/* replaces utilslib.compute_raydirs_forward — utils.cpp:46-82 (kernel utils_kernel.cu:11-51).
 * viewpos [N,3], viewrot [N,3,3], focal [N,2], princpt [N,2], pixelcoords [N,H,W,2] or NULL (integer grid),
 * outputs raypos/raydir [N,H,W,3], tminmax [N,H,W,2]. */
int gb_compute_raydirs_fwd(int N, int H, int W, const float* viewpos, const float* viewrot, const float* focal,
                           const float* princpt, const float* pixelcoords, float volradius, float* raypos,
                           float* raydir, float* tminmax, void* stream);
/* replaces utilslib.compute_raydirs_backward — utils.cpp:84-132: the reference kernel is an empty stub. */
int gb_compute_raydirs_bwd(void);

/* ---------------------------------------------------------------- mvpraymarchlib (extensions/mvpraymarch) */

/* replaces mvpraymarchlib.compute_aabb — mvpraymarch.cpp (compute_aabb) -> bvh.cu:157-201,249-294.
 * Tree arrays as built by mvpraymarch.py:44-82; nodeaabb [N,2K-1,2,3] out; workspace of
 * gb_mvp_aabb_workspace_bytes(N,K) bytes replaces the reference's per-call cudaMalloc. */
size_t gb_mvp_aabb_workspace_bytes(int N, int K);
int gb_mvp_compute_aabb(int N, int K, const float* primpos, const float* primrot, const float* primscale,
                        const int32_t* sortedobjid, const int32_t* nodechildren, const int32_t* nodeparent,
                        float* nodeaabb, void* workspace, void* stream);

/* march formulation for algo 0 without the shadow splat: bit 0 / bit 1 = lane-compacted sampling queue in the forward /
 * backward march (inside-the-box (ray, primitive) pairs are enqueued, sampled 32 at a time with every lane busy, applied in
 * the original order); default 2: the backward only (measured: backward 9.9 -> 8.3 ms at config 4, forward slower
 * with the queue).  GOLIATH_B200_RAYMARCH=legacy|queue-fwd|queue-bwd|queue. */
int gb_get_raymarch_mode(void);
void gb_set_raymarch_mode(int mode);

/* replaces mvpraymarchlib.raymarch_forward — mvpraymarch.cpp:179-283 -> mvpraymarch_kernel.cu:41-130.
 * template [N,K,TD,TH,TW,4] channels-last; warp [N,K,WD,WH,WW,3] or NULL (algo 0); rayrgba [N,H,W,4] out;
 * raysat [N,H,W,3] out or NULL; shadow [N,K,TD,TH,TW,2] accumulated or NULL.  The arguments the reference
 * accepts and ignores (sortboxes, maxhitboxes, synchitboxes, chlast, accum, termthresh, griddim, SURVEY.md §0.9)
 * are handled by the Python binding and are not part of the ABI. */
int gb_mvp_raymarch_fwd(int N, int H, int W, int K, const float* raypos, const float* raydir, float stepsize,
                        const float* tminmax, const float* nodeaabb, const float* primpos, const float* primrot,
                        const float* primscale, int TD, int TH, int TW, const float* tplate, int WD, int WH, int WW,
                        const float* warp, float* rayrgba, float* raysat, float* shadow, int algo, float fadescale,
                        float fadeexp, int blocksizex, int blocksizey, void* stream);

/* replaces mvpraymarchlib.raymarch_backward — mvpraymarch.cpp:285-399 -> mvpraymarch_kernel.cu:132-221.
 * Gradient buffers are accumulated into (the caller zero-fills them, mvpraymarch.py:256-263). */
int gb_mvp_raymarch_bwd(int N, int H, int W, int K, const float* raypos, const float* raydir, float stepsize,
                        const float* tminmax, const float* nodeaabb, const float* primpos, const float* primrot,
                        const float* primscale, int TD, int TH, int TW, const float* tplate, int WD, int WH, int WW,
                        const float* warp, const float* raysat, const float* grad_rayrgba, float* grad_primpos,
                        float* grad_primrot, float* grad_primscale, float* grad_tplate, float* grad_warp, int algo,
                        float fadescale, float fadeexp, int blocksizex, int blocksizey, void* stream);

/* ---------------------------------------------------------------- RGCA decoder heads (row R2) */

/* replaces the eager PyTorch block ca_code/models/rgca.py:506-546 (Gaussian heads, SH diffuse, reflection
 * direction); there is no native boundary in the reference, the Python mirror is goliath_b200.rgca_heads.
 * f_vnocond [B,125,G], f_vcond [B,4,G], postex / tn [B,3,G] planes (G = H*W), albedo [G,3], light_sh [B,3,81],
 * campos [B,3].  Outputs [B,G,3] except primqvec [B,G,4] and opacity / sigma / spec_vis [B,G]; shsum [B,G,3] is
 * saved for the backward. */
int gb_rgca_heads_fwd(int B, int G, const float* f_vnocond, const float* f_vcond, const float* postex, const float* tn,
                      const float* albedo, const float* light_sh, const float* campos, float scale_lo, float scale_hi,
                      float* primpos, float* primqvec, float* primscale, float* primscale_preclip, float* opacity,
                      float* sigma, float* spec_vis, float* spec_dnml, float* spec_nml, float* diff_color,
                      float* ref_dirs, float* primnmlbase, float* shsum, const float* light_sh2, float* shsum2,
                      void* stream);
/* light_sh2 [B,3,81] / shsum2 [B,G,3] (both NULL or both set): a second light-SH table evaluated in the same pass over the
 * 113 diffuse planes — the training-mode random back light `diff_color_rand` of rgca.py:590-616 (no albedo, unclamped). */

/* backward of the above; upstream gradients may be NULL; g_albedo is [B,G,3] (summed over B by the caller);
 * light_sh2 / g_shsum2: the second table and the upstream gradient of shsum2 (both NULL when unused). */
int gb_rgca_heads_bwd(int B, int G, const float* f_vnocond, const float* f_vcond, const float* postex, const float* tn,
                      const float* albedo, const float* light_sh, const float* campos, float scale_lo, float scale_hi,
                      const float* shsum, const float* g_primpos, const float* g_primqvec, const float* g_primscale,
                      const float* g_primscale_preclip, const float* g_opacity, const float* g_sigma,
                      const float* g_spec_vis, const float* g_spec_dnml, const float* g_spec_nml,
                      const float* g_diff_color, const float* g_ref_dirs, const float* g_primnmlbase, float* g_f_vnocond,
                      float* g_f_vcond, float* g_postex, float* g_tn, float* g_albedo, const float* light_sh2,
                      const float* g_shsum2, void* stream);

/* ---------------------------------------------------------------- mesh front end of the decoders (section 8f-4) */

/* replaces vert_normals (ca_code/utils/geom.py:327-346): v [B,V,3], vi [F,3] -> vn [B,V,3]; acc [B,V,3] = scratch
 * zero-filled by the caller (sum of the unit face normals per vertex), kept for the backward. */
int gb_vert_normals_fwd(int B, int V, int F, const float* v, const int32_t* vi, float eps, float* acc, float* vn, void* stream);
/* g_vn -> g_v [B,V,3] (zero-filled by the caller, accumulated); g_acc [B,V,3] scratch. */
int gb_vert_normals_bwd(int B, int V, int F, const float* v, const int32_t* vi, float eps, const float* acc, const float* g_vn,
                        float* g_acc, float* g_v, void* stream);
/* replaces values_to_uv (ca_code/utils/geom.py:308-324, GeometryModule.to_uv): values [B,V,C], index [T,3] int32 (-1 =
 * uncovered), bary [T,3] -> out [B,C,T] with T = uv_size^2. */
int gb_values_to_uv_fwd(int B, int V, int C, int64_t T, const float* values, const int32_t* index, const float* bary, float* out,
                        void* stream);
/* g_out [B,C,T] -> g_values [B,V,C] (zero-filled by the caller, accumulated). */
int gb_values_to_uv_bwd(int B, int V, int C, int64_t T, const int32_t* index, const float* bary, const float* g_out,
                        float* g_values, void* stream);

/* ---------------------------------------------------------------- gradient hygiene + clip + Adam (section 8f-3) */

/* replaces ca_code/utils/train.py:209-215 around the optimizer of config/*.yml (torch.optim.Adam / AdamW): zero the NaN /
 * Inf gradient entries, clip_grad_norm_(params, max_norm), optimizer.step().  rows: device array of 56-byte records
 * {float* p, g, m, v; int64 numel; float lr, wd; int32 missed, pad} (g == NULL: parameter skipped; missed = steps it sat out); chunks: device (tensor, chunk) int32
 * pairs covering every tensor in steps of gb_optim_chunk_elems() elements. */
int gb_optim_chunk_elems(void);
int gb_optim_row_bytes(void);
/* non-finite gradient entries -> 0 in place; *sqnorm (device fp64, zero-filled by the caller) += sum of squares. */
int gb_grad_sanitize_sqnorm(const void* rows, const int32_t* chunks, int n_chunks, double* sqnorm, void* stream);
/* Adam (adamw = 0, L2 weight decay) or AdamW (adamw = 1) step; gradients scaled by clamp(max_norm / (sqrt(*sqnorm) + 1e-6),
 * max = 1) when sqnorm != NULL and max_norm > 0; bias corrections 1 - beta^(step - row.missed); write_grads = 1 stores the clipped
 * gradients back (what clip_grad_norm_ leaves in p.grad). */
int gb_adam_step(const void* rows, const int32_t* chunks, int n_chunks, const double* sqnorm, float max_norm, float beta1,
                 float beta2, float eps, int step, int adamw, int write_grads, void* stream);

/* ---------------------------------------------------------------- post-render chain + photometric losses (section 8f-2) */

/* replaces CalV5.forward (ca_code/nn/color_cal.py:211-241), the background composite of rgca.AutoEncoder.forward
 * (ca_code/models/rgca.py:226-230) and LearnableBlur.forward (ca_code/nn/dof_cal.py:44-56; torchvision gaussian_blur 3x3 /
 * 7x7, reflect padding): pred = blur(cal(rgb) + (1 - alpha) * bg).  rgb / bg / pred [B,3,H,W], alpha [B,1,H,W], cal_w / cal_b /
 * blur_w [B,3] (blur_w = softmax-ed weights), grey [B] int32.  Stages with NULL tensors are skipped. */
int gb_post_render_fwd(int B, int H, int W, const float* rgb, const float* alpha, const float* bg, const float* cal_w,
                       const float* cal_b, const int32_t* grey, const float* blur_w, float* pred, void* stream);
/* g_pred -> g_rgb (overwritten); g_cal_w / g_cal_b / g_blur_w [B,3] accumulated (zero-filled by the caller, may be NULL). */
int gb_post_render_bwd(int B, int H, int W, const float* rgb, const float* alpha, const float* bg, const float* cal_w,
                       const float* cal_b, const int32_t* grey, const float* blur_w, const float* g_pred, float* g_rgb,
                       float* g_cal_w, float* g_cal_b, float* g_blur_w, void* stream);
/* replaces rgb_l1 and rgb_ssim (ca_code/loss/__init__.py:391-410, 479-494 over ca_code/utils/ssim.py:25-63): sums [3] fp64
 * (zero-filled by the caller) = sum |(pred - target) * mask|, sum ssim_map * mask, sum of the mask over 3 channels;
 * d_mu / d_pp / d_tp [B,3,H,W] are kept for the backward. */
int gb_ssim_l1_fwd(int B, int H, int W, const float* pred, const float* target, const float* mask, float* d_mu, float* d_pp,
                   float* d_tp, double* sums, void* stream);
/* gradient of l1_weight * rgb_l1 + ssim_weight * rgb_ssim w.r.t. pred, times *g_loss (device scalar, NULL = 1). */
int gb_ssim_l1_bwd(int B, int H, int W, const float* pred, const float* target, const float* mask, const float* d_mu,
                   const float* d_pp, const float* d_tp, const double* sums, const float* g_loss, float l1_weight,
                   float ssim_weight, float* g_pred, void* stream);

/* replaces the environment-map specular branch of rgca.PrimDecoder.forward (ca_code/models/rgca.py:548-556):
 * einsum("bxy,bny->bnx", lightrot, ref_dirs) -> dir2uv (ca_code/utils/envmap.py:284-292) -> mipmap_grid_sample of the
 * pre-convolved pyramid at level sigma * level_scale (ca_code/utils/mipmap_sampler.py:13-66: bilinear, border padding,
 * align_corners=False, two adjacent levels blended by the fractional level) -> clamp(max=1) * spec_vis.
 * levels: q (1..8) device pointers to [B,3,H_l,W_l] fp32 (the array itself in HOST memory); level_hw: q (H, W) pairs
 * (host).  ref_dirs [B,G,3], sigma [B,G], spec_vis [B,G], lightrot [B,3,3] -> spec [B,G,3]. */
int gb_envmap_spec_fwd(int B, int G, int q, const float* const* levels, const int32_t* level_hw, const float* ref_dirs,
                       const float* sigma, const float* spec_vis, const float* lightrot, float level_scale, float* spec,
                       void* stream);
/* g_spec [B,G,3] -> g_ref_dirs [B,G,3], g_spec_vis [B,G] (overwritten); no gradient for sigma (the level is picked
 * under no_grad upstream) nor for the environment map. */
int gb_envmap_spec_bwd(int B, int G, int q, const float* const* levels, const int32_t* level_hw, const float* ref_dirs,
                       const float* sigma, const float* spec_vis, const float* lightrot, float level_scale,
                       const float* g_spec, float* g_ref_dirs, float* g_spec_vis, void* stream);

/* replaces rotate_envmap_mat (ca_code/utils/envmap.py:141-166), batched over B: texel grid
 * theta = (i + 0.5) * 3.1415926 / He, phi = (j - We//2 + 0.5) * 3.1415926 * 2 / We, vec = (sin t sin p, cos t, sin t cos p),
 * vec @ R^T (= R vec) clamped to [-1, 1] per component, dir2uv (np.pi), bilinear grid_sample (border padding,
 * align_corners=False).  image / out [B,3,He,We], rot_mat [B,3,3] (row-major R). */
int gb_envmap_rotate(int B, int He, int We, const float* image, const float* rot_mat, float* out, void* stream);
/* replaces compose_envmap (ca_code/utils/envmap.py:325-345) with envmap_to_image (:169-227, focal_scale 0.2, blurbg,
 * no fisheye D) and envmap_to_mirrorball (:230-248, 200x200):
 *   rays d = ((x - K[0,2]) / (0.2 K[0,0]), (y - K[1,2]) / (0.2 K[1,1]), 1), rotated R^T d (einsum "bxy,bhwx->bhwy" with
 *   R = Rt[:3,:3]), normalised, dir2uv; bicubic grid_sample (A = -0.75, border padding applied to each of the 16 taps,
 *   align_corners=True); the 101x101 blur k(x)k / sum(k(x)k), k = exp(-linspace(-4, 4, 101)^2), zero padding 50, run as
 *   two separable 101-tap passes; bg' = render + (1 - alpha) * clamp(bg, 0, 1); out = (1 - m) * bg' + m * mirror in the
 *   bottom-right 200x200 corner, m = (zsq < 1) on torch's linspace(-1, 1, 200) grid, mirror colour unclamped.
 * acos is taken without a clamp, as the reference does: where rounding (or a non-orthonormal Rt) pushes the y
 * component past +-1, the sample is NaN, the blur spreads it over the 101x101 neighbourhood, and the mirror ball
 * (whose reflected directions are not normalised) turns NaN at that pixel and, through m * NaN, at masked-out
 * pixels of the corner too; clamp keeps NaN.
 * render / out [B,3,H,W], alpha [B,1,H,W], envbg [B,3,He,We], K [B,3,3], Rt [B,rt_rows,rt_cols] (rt_rows, rt_cols >= 3),
 * all in device memory (no host sync); hblur [B,3,H,W] scratch.  H, W >= 200. */
int gb_envmap_compose_fwd(int B, int H, int W, int He, int We, const float* render, const float* alpha,
                          const float* envbg, const float* K, const float* Rt, int rt_rows, int rt_cols, float* hblur,
                          float* out, void* stream);
/* the only gradient of compose_envmap (alpha detached, envbg / K / Rt data): g_render = (1 - m) * g_out [B,3,H,W]. */
int gb_envmap_compose_bwd(int B, int H, int W, const float* g_out, float* g_render, void* stream);
/* replaces prefilterEnvmapSG (ca_code/utils/envmap.py:305-323) with importance_sample_sg (:251-281, the pdf not computed)
 * and sample_uv (:295-302), for q (1..8) levels in one launch: out[l] [B,3,H,W] = mean over num_samples of the bilinear
 * lookup (border padding, align_corners=False) of env_tex[l] [B,3,He,We] along normalize(t Hx + b Hy + n Hz), n = v[l]
 * [B,3,H,W], up = (0,0,1) where n_z < 0.999 else (1,0,0), t = normalize(up x n), b = n x t, H = (cos phi sin theta,
 * sin phi sin theta, cos theta), phi = 2 pi xi0, theta = sqrt(2) sigma erfinv(xi1 erf(pi / (sqrt(2) sigma))).
 * dir2uv takes acos without a clamp, as the reference does: where rounding pushes the normalised y past +-1 the v
 * coordinate is NaN, which grid_sample's border clip (and this kernel) turns into 0, so that sample reads the first
 * texel row.  xi: NULL, or q device pointers to [num_samples,B,2,H,W] (the reference's th.rand_like(v[:, :2]) draws);
 * with NULL, xi comes from a counter-based Philox4x32-10 stream keyed by seed at counter (sample pair, texel, item, l),
 * and the per-texel sum runs in a fixed order, so a seed gives bit-identical output.
 * level_hw: q x (H, W, He, We) and sigma [q] (> 0) in host memory; v / env_tex / xi / out: host arrays of device
 * pointers. */
int gb_envmap_prefilter_sg(int B, int q, const int32_t* level_hw, const float* sigma, const float* const* v,
                           const float* const* env_tex, const float* const* xi, int num_samples, unsigned long long seed,
                           float* const* out, void* stream);
/* replaces the per-item loop of EnvSpinDecorator.forward (ca_code/utils/light_decorator.py:111-149), batched over B:
 *   lightrot [B,3,3] = rvec_to_R((0, angles[b], 0)) (ca_code/utils/envmap.py:20-50, fp32; angle 0 gives I);
 *   envbg [B,3,He,We] = rotate_envmap_mat(image, lightrot[b]) (gb_envmap_rotate) / perc90 * 255 / 255;
 *   the 16x32 antialiased bilinear downsample of the rotated probe (torch's _upsample_bilinear2d_aa weights, horizontal
 *   pass first into hpass [B,3,He,32] scratch);
 *   envmap [B,3,16,32] = env_scale * down / sum(down * sin((row + 0.5) pi / 16)) over channels and texels;
 *   light_intensity [B,512,3] = envmap[b].view(3, -1).t(); norm_scale [B] = env_scale / that sum.
 * angles [B] in host memory (2 pi index / cycle); image [3,He,We] the static probe; perc90 > 0 its 90th percentile;
 * He >= 16, 32 <= We <= 3072.  No host sync, no copy. */
int gb_envmap_spin_table(int B, int He, int We, const float* angles, const float* image, float perc90, float env_scale,
                         float* lightrot, float* envbg, float* hpass, float* envmap, float* light_intensity,
                         float* norm_scale, void* stream);

/* replaces the per-view post-processing of rgca.AutoEncoder.render (ca_code/models/rgca.py:136-151, with
 * render_gsplat.py:79-108): colour HWC -> CHW, alpha = 1 - final_T (detached), depth / alpha.clamp(0.05, 1).
 * out4 [H,W,4] = rgb + depth-as-colour, alpha [H,W] -> rgb [3,H,W], alpha_img [1,H,W], depth [1,H,W]. */
int gb_render_finish_fwd(int img_h, int img_w, const float* out4, const float* alpha, float* rgb, float* alpha_img,
                         float* depth, void* stream);
/* g_rgb / g_depth may be NULL; g_out4 [H,W,4] is written. */
int gb_render_finish_bwd(int img_h, int img_w, const float* alpha, const float* g_rgb, const float* g_depth,
                         float* g_out4, void* stream);

/* fused shade + compose: replaces F.normalize (extensions/sgutils/sgutils.py:74-75) + evaluate_gaussian + the colour
 * composition of ca_code/models/rgca.py:557-575 (`spec * spec_vis`, `diff.clamp(0) + spec`, `.clamp(0)`) with one kernel
 * each way.  lobe_dirs are the UN-normalised reflection directions [N,D,3]; diff_color [N,D,3], spec_vis [N,D];
 * color [N,D,3] out (its sign bit keeps the pre-clamp sign for the backward); spec_color [N,D,3] out or NULL. */
int gb_sg_shade_compose_fwd(const float* lobe_dirs, const float* lobe_sigmas, const float* light_values,
                            const float* light_pts, const float* prim_pts, const int32_t* n_lights,
                            const float* diff_color, const float* spec_vis, float* color, float* spec_color, int N,
                            int D, int L, int w_type, void* stream);
/* backward: color = the forward's output; g_spec_color may be NULL; g_dirs / g_sigmas / g_diff / g_vis are written,
 * g_light_values (nullable) is accumulated into (caller zeroes it). */
int gb_sg_shade_compose_bwd(const float* lobe_dirs, const float* lobe_sigmas, const float* light_values,
                            const float* light_pts, const float* prim_pts, const int32_t* n_lights,
                            const float* diff_color, const float* spec_vis, const float* color, const float* g_color,
                            const float* g_spec_color, float* g_dirs, float* g_sigmas, float* g_diff, float* g_vis,
                            float* g_light_values, int N, int D, int L, int w_type, void* stream);

/* ---------------------------------------------------------------- decoder layers (rows R1 / R8) */

/* replaces conv_transpose2d + untied-bias add (ca_code/nn/layers.py:380-396) + the LeakyReLU that follows it in
 * make_conv_trans (layers.py:27-47) for k=4, s=2, p=1, with the weight-norm scale folded in:
 * out = act(scale[co] * convT(x, v) + bias).  x [B,Cin,Hi,Wi], v [Cin,Cout,4,4], scale [Cout] = g / ||v||_F,
 * bias [Cout,2Hi,2Wi] or NULL, out [B,Cout,2Hi,2Wi]; apply_act != 0 applies LeakyReLU(slope). */
int gb_deconv4x4s2_wnub_fwd(int B, int Cin, int Cout, int Hi, int Wi, const float* x, const float* v,
                            const float* scale, const float* bias, float slope, int apply_act, float* out,
                            void* stream);

/* backward of the above (replaces the cuDNN backward-data / backward-filter calls autograd makes for
 * layers.py:380-396).  gz [B,Cout,2Hi,2Wi] scratch when apply_act, else unused (may be NULL); g_bias [Cout,2Hi,2Wi]
 * written, or NULL; gx [B,Cin,Hi,Wi] or NULL; gw [Cin,Cout,4,4] = dL/d(effective weight at unit scale) written (the
 * caller applies the weight-norm chain rule).  Every sum runs in a fixed order (no float atomics), so the gradients
 * are bitwise repeatable.  `workspace`: gb_deconv4x4s2_wnub_bwd_workspace_bytes(B, Cin, Cout, Hi, Wi) bytes. */
size_t gb_deconv4x4s2_wnub_bwd_workspace_bytes(int B, int Cin, int Cout, int Hi, int Wi);
int gb_deconv4x4s2_wnub_bwd(int B, int Cin, int Cout, int Hi, int Wi, const float* x, const float* v,
                            const float* scale, const float* out, const float* gout, float slope, int apply_act,
                            float* gz, float* g_bias, float* gx, float* gw, void* workspace, void* stream);

/* replaces conv2d + untied-bias add (ca_code/nn/layers.py:276-327) + the LeakyReLU that follows each
 * la.Conv2dWNUB(cin, cout, h, w, 4, 2, 1) of the RGCA texture encoder (ca_code/models/rgca.py:281-298) for k=4, s=2,
 * p=1, with the weight-norm scale folded in: out = act(scale[co] * conv(x, v) + bias).  x [B,Cin,2Ho,2Wo],
 * v [Cout,Cin,4,4], scale [Cout] = g / ||v||_F, bias [Cout,Ho,Wo] or NULL, out [B,Cout,Ho,Wo]; apply_act != 0 applies
 * LeakyReLU(slope).  Runs on the kernels of gb_deconv4x4s2_wnub_bwd with the two sides of the layer exchanged. */
int gb_conv4x4s2_wnub_fwd(int B, int Cin, int Cout, int Ho, int Wo, const float* x, const float* v,
                          const float* scale, const float* bias, float slope, int apply_act, float* out, void* stream);

/* backward of the above, with the conventions of gb_deconv4x4s2_wnub_bwd.  gz [B,Cout,Ho,Wo] scratch when
 * apply_act, else unused; g_bias [Cout,Ho,Wo] written, or NULL; gx [B,Cin,2Ho,2Wo] or NULL; gw [Cout,Cin,4,4] =
 * dL/d(effective weight at unit scale) written (the caller applies the weight-norm chain rule).  Bitwise repeatable.
 * `workspace`: gb_conv4x4s2_wnub_bwd_workspace_bytes(B, Cin, Cout, Ho, Wo) bytes. */
size_t gb_conv4x4s2_wnub_bwd_workspace_bytes(int B, int Cin, int Cout, int Ho, int Wo);
int gb_conv4x4s2_wnub_bwd(int B, int Cin, int Cout, int Ho, int Wo, const float* x, const float* v,
                          const float* scale, const float* out, const float* gout, float slope, int apply_act,
                          float* gz, float* g_bias, float* gx, float* gw, void* workspace, void* stream);

/* ---- tensor-core (wgmma + TMA) forward of the same layer, inference path; Cin_pad % 32 == 0,
 * Cout % 16 == 0, 16 <= Cout <= 256.  Activations are NHWC split into a tf32 "hi" part and the fp32 remainder "lo"
 * (3xTF32 accumulation keeps the 1e-4 bar).  Same reference lines as gb_deconv4x4s2_wnub_fwd.
 * v may be NULL when w_scratch still holds the matrices prepared by an earlier call with the same weight_v
 * (inference with frozen parameters). */
size_t gb_deconv_tc_weight_bytes(int Cin_pad, int Cout);
int gb_nchw_to_nhwc_split(int B, int C, int Cpad, int H, int W, const float* x, float* hi, float* lo, void* stream);
int gb_deconv4x4s2_tc_fwd(int B, int Cin, int Cin_pad, int Cout, int Hi, int Wi, const float* x_hi, const float* x_lo,
                          const float* v, float* w_scratch, const float* scale, const float* bias, float slope,
                          int apply_act, float* out_hi, float* out_lo, int ldc, float* out_nchw, void* stream);

/* ---------------------------------------------------------------- hand-MVP decoders (row R8) */

/* replaces conv2d + bias add (+ LeakyReLU) of la.Conv2dWNUB / Conv2dWN (ca_code/nn/layers.py:276-327,468-472;
 * users: hand_mvp.py:297-321 TransDecoder, hand_mvp.py:269-294 PoseEncoder via blocks.py:232-280 ConvBlock, and
 * th.split + la.Conv2dWNUB of mesh_vae.py:615-621, verts_conv / tex_conv on a channel slice read in place), stride 1,
 * K = 1 or 3, padding (K-1)/2, with the weight-norm scale folded in: out = act(scale[co] * conv(x, v) + bias).
 * x [B,Cin,H,W] with items x_bs >= Cin*H*W floats apart; v [Cout,Cin,K,K], scale [Cout] = g / ||v||_F; bias_mode 0 none,
 * 1 tied [Cout], 2 untied [Cout,H,W]. */
int gb_conv2d_wnub_fwd(int B, int Cin, int Cout, int H, int W, int K, const float* x, long long x_bs, const float* v,
                       const float* scale, const float* bias, int bias_mode, float slope, int apply_act, float* out,
                       void* stream);

/* replaces the autograd graph of the layer above.  gz [B,Cout,H,W] scratch when apply_act, else unused (may be NULL);
 * g_bias: [Cout,H,W] (mode 2) or [Cout] (mode 1) written, or NULL; gx [B,Cin,H,W] with items x_bs floats apart, or
 * NULL; gw [Cout,Cin,K,K] = dL/d(effective weight at unit scale) written (the caller applies the weight-norm chain
 * rule).  Every sum runs in a fixed order (no float atomics), so the gradients are bitwise repeatable.
 * `workspace`: gb_conv2d_wnub_bwd_workspace_bytes(B, Cin, Cout, H, W, K) bytes. */
size_t gb_conv2d_wnub_bwd_workspace_bytes(int B, int Cin, int Cout, int H, int W, int K);
int gb_conv2d_wnub_bwd(int B, int Cin, int Cout, int H, int W, int K, const float* x, long long x_bs, const float* v,
                       const float* scale, const float* out, const float* gout, float slope, int apply_act,
                       int bias_mode, float* gz, float* g_bias, float* gx, float* gw, void* workspace, void* stream);

/* replaces the slab -> primitive-template sequence: relu(25*rgb+100) (hand_mvp.py:472), relu(alpha) (:434),
 * cat/view/permute/reshape (hand_mvp.py:172-185) and the valid-primitive gather (ca_code/utils/render_raymarcher.py:44-46)
 * with one pass.  rgb [B,PZ,3,U,U], alpha [B,PZ,1,U,U]; prim_slot [(U/PSY)*(U/PSX)] i32 (slot of a primitive in the
 * output, -1 = dropped) or NULL; tpl [B,Kout,PZ,PSY,PSX,4].  rgb_mul/rgb_add/apply_relu carry the output activation
 * (1, 0, 0 for a plain re-layout of already-activated slabs). */
int gb_mvp_slab_to_prims_fwd(int B, int PZ, int U, int PSX, int PSY, int Kout, const float* rgb, const float* alpha,
                             const int* prim_slot, float rgb_mul, float rgb_add, int apply_relu, float* tpl,
                             void* stream);
int gb_mvp_slab_to_prims_bwd(int B, int PZ, int U, int PSX, int PSY, int Kout, const float* rgb, const float* alpha,
                             const int* prim_slot, float rgb_mul, float rgb_add, int apply_relu, const float* g_tpl,
                             float* g_rgb, float* g_alpha, void* stream);

/* replaces TransDecoder's head scaling (hand_mvp.py:317-321) + GeomDecoder's transform composition
 * (hand_mvp.py:410-425, axisangle_to_matrix :477-510).  dec [B,9,K] (dec0 output viewed [B,9,64*64]);
 * posbase [B,K,3], rotbase [B,K,3,3]; zero_delta = the `iteration < primposstart` warm start (:412-415). */
int gb_mvp_prim_transform_fwd(int B, int K, const float* dec, const float* posbase, const float* rotbase,
                              float prim_scale, int zero_delta, float* primpos, float* primrot, float* primscale,
                              void* stream);
int gb_mvp_prim_transform_bwd(int B, int K, const float* dec, const float* posbase, const float* rotbase,
                              float prim_scale, int zero_delta, const float* g_primpos, const float* g_primrot,
                              const float* g_primscale, float* g_dec, void* stream);

/* replaces make_postex (ca_code/utils/geom.py:515-520) and compute_tbn (geom.py:355-397) as hand_mvp.GeomDecoder.forward
 * calls them (hand_mvp.py:393-408), and compute_view_cos (geom.py:349-352) + values_to_uv (geom.py:308-324) as
 * hand_mvp.AutoEncoder.forward calls them (hand_mvp.py:230-236).  One thread per (item, texel) on the posed vertices
 * verts [B,V,3]; vidx / vtidx / bary [T,3] (int32, int32, fp32), vt [NT,2].  Outputs (each may be NULL):
 *   posbase [B,T,3] = b0 v[i0] + b1 v[i1] + b2 v[i2];
 *   rotbase [B,T,3,3] with the columns T, B, N of compute_tbn: f = 1/det of the UV edges, taken without a guard (a
 *   degenerate UV triangle gives NaN, as in the reference), F.normalize with eps 1e-12, bitangent = normalize(T x N);
 *   view_cos [B,T] = sum_k b_k <normalize(vn[i_k]), normalize(v[i_k] - campos[b])>, 0 where any index is -1;
 *   vn [B,V,3] comes from gb_vert_normals_fwd, campos [B,3].
 * A negative index in the frame outputs selects from the end, as torch's indexing does.  vtidx / vt are needed for
 * rotbase, vn / campos for view_cos. */
int gb_mvp_prim_frames_fwd(int B, int V, int NT, int T, const float* verts, const int32_t* vidx, const int32_t* vtidx,
                           const float* bary, const float* vt, const float* vn, const float* campos, float* posbase,
                           float* rotbase, float* view_cos, void* stream);

/* ---------------------------------------------------------------- linear blend skinning (row R8') */

/* Largest joint count gb_lbs_skeleton_fwd accepts: one CTA keeps every joint's state (8 floats) in shared memory. */
int gb_lbs_max_joints(void);

/* replaces ParameterTransform.forward + solve_skeleton_state + states_to_matrix (ca_code/utils/lbs.py:39-46,340-429)
 * as LinearBlendSkinning.forward runs them (lbs.py:308-337), with the quaternion operations of
 * ca_code/utils/quaternion.py:178-320.  One CTA per item b:
 *   jp = transform [7J,P+S] . cat(motion[b] [P], scale[b] [S]) + transform_offsets [7J];
 *   per joint: lt = jp[0:3] + joint_offset, lr = joint_rotation (x) fromXYZ(jp[3:6]), ls = 2^jp[6];
 *   per joint with parent p, level by level: q = q_p (x) lr, t = rot(q_p, lt s_p) + t_p, s = s_p ls.
 * scale rows are scale_stride floats apart (0 = one row for every item).  parents [J] int32 (-1 = root, parent < j);
 * level_order [J] lists the joints level by level (roots first), level_start [n_levels+1] the level boundaries.
 * bind_state [J,8] -> mats [B,J,3,4] (states_to_matrix); states [B,J,8] (t, q, s) is written when not NULL.
 * J > gb_lbs_max_joints() returns cudaErrorInvalidValue. */
int gb_lbs_skeleton_fwd(int B, int J, int P, int S, const float* motion, const float* scale, int scale_stride,
                        const float* transform, const float* transform_offsets, const float* joint_offset,
                        const float* joint_rotation, const int32_t* parents, const int32_t* level_order,
                        const int32_t* level_start, int n_levels, const float* bind_state, float* mats, float* states,
                        void* stream);

/* replaces LinearBlendSkinning.skinning (lbs.py:226-254) and the template add / global scaling of LBSModule.pose
 * (lbs.py:725-731): out [B,V,3] = gs * sum_{k<8} w_k mats[b, idx_k] [verts + templ; 1], slots summed in order.
 * verts [vb,V,3] with vb = 1 or B; templ [V,3] or NULL (zero); skin_indices [V,8] int32, skin_weights [V,8];
 * global_scaling [3] or NULL (one). */
int gb_lbs_skin_fwd(int B, int V, int J, int vb, const float* mats, const float* verts, const float* templ,
                    const int32_t* skin_indices, const float* skin_weights, const float* global_scaling, float* out,
                    void* stream);
/* gradient w.r.t. verts only: g_verts [vb,V,3] (written) = sum_k w_k mats[b, idx_k][:, :3]^T (gs * g_out[b]); a batch-1
 * input sums b = 0..B-1 in order inside one thread, so the result is deterministic. */
int gb_lbs_skin_bwd(int B, int V, int J, int vb, const float* mats, const int32_t* skin_indices,
                    const float* skin_weights, const float* global_scaling, const float* g_out, float* g_verts,
                    void* stream);

/* replaces LinearBlendSkinning.unskinning (lbs.py:273-306: a [B,V,4,4] blended matrix and inverse() in a Python loop
 * over the batch) and the scaling / template of LBSModule.unpose (lbs.py:733-739):
 *   out [B,V,3] = (sum_{k<8} w_k mats[b, idx_k])^-1 [verts / gs; 1] - templ.
 * The blended [3,4] matrix [A | t] is inverted as an affine map in registers (adjugate / determinant in double, then
 * A^-1 (x - t)); the reference's fourth row is (0,0,0,1), so this is its 4x4 inverse.  det(A) == 0 writes NaN for that
 * vertex.  Arguments as gb_lbs_skin_fwd; forward only. */
int gb_lbs_unskin_fwd(int B, int V, int J, int vb, const float* mats, const float* verts, const float* templ,
                      const int32_t* skin_indices, const float* skin_weights, const float* global_scaling, float* out,
                      void* stream);

/* ---------------------------------------------------------------- relightable hand teacher (row R8'') */

/* replaces the deep shadow march of OLATRGBDecoder.forward_rgb (hand_teacher_mvp.py:274-358: the expanded [B*L, K,
 * TD, TH, TW, 4] template through mvpraymarch(with_shadow=True)).  Forward only, arithmetic of the shadow-splatting
 * forward march without its rgb.  N = B*L light views; view n reads the transforms [B,K,3] / [B,K,3,3] / [B,K,3] and
 * bounds [B,2K-1,2,3] (gb_mvp_compute_aabb with N = B) of item n / L and samples the alpha slab [B,TD,U,U] in place
 * (K = (U/TW)*(U/TH) primitives, row-major), times valid [K] (NULL = all valid).  shadow [N,K,TD,TH,TW,2] is
 * accumulated into (the caller zero-fills it); nothing else is written. */
int gb_mvp_shadow_march(int N, int L, int H, int W, int K, const float* raypos, const float* raydir, float stepsize,
                        const float* tminmax, const float* nodeaabb, const float* primpos, const float* primrot,
                        const float* primscale, int TD, int TH, int TW, int U, const float* alpha_slab,
                        const float* valid, float* shadow, float fadescale, float fadeexp, int blocksizex,
                        int blocksizey, void* stream);

/* replaces the no_grad feature block of OLATRGBDecoder.forward_rgb (hand_teacher_mvp.py:359-439): U-Net input
 * feat [B*L,7*TD,U,U] (light vector, view direction in the primitive frame, 1 - shadow), primshadow [B,TD,3,U,U]
 * (the light mean of the normalised shadow, added when accumulate) and, when not NULL, the normalised shadow
 * shadow_feat [B*L,TD,U,U].  Transforms in world units, light_pos [B,L,3], campos [B,3], shadow from
 * gb_mvp_shadow_march. */
int gb_olat_features(int B, int L, int K, int TD, int TH, int TW, int U, float volradius, const float* primpos,
                     const float* primrot, const float* primscale, const float* valid, const float* light_pos,
                     const float* campos, const float* shadow, float* feat, float* primshadow, int accumulate,
                     float* shadow_feat, void* stream);

/* replaces the OLAT compose of OLATRGBDecoder.forward_rgb (hand_teacher_mvp.py:468-479): rgb [B,Z,3,U,U] (added when
 * accumulate) = sum_l s relu(25 t_c + 100) I[b,l,c] over tex [B*L,4Z,U,U] viewed [B,L,Z,4,U,U], s = sigmoid(t_0) or
 * shadow_feat [B*L,Z,U,U] when not NULL; texolat [B,L,Z,3,U,U] = 25 t_c + 100 when not NULL. */
int gb_olat_compose_fwd(int B, int L, int Z, int U, const float* tex, const float* intensity, const float* shadow_feat,
                        float* rgb, int accumulate, float* texolat, void* stream);
/* g_tex [B*L,4Z,U,U] (written) from g_rgb [B,Z,3,U,U] and g_texolat [B,L,Z,3,U,U] or NULL; t_0 gets zero when
 * shadow_feat is given. */
int gb_olat_compose_bwd(int B, int L, int Z, int U, const float* tex, const float* intensity, const float* shadow_feat,
                        const float* g_rgb, const float* g_texolat, float* g_tex, void* stream);

/* ---------------------------------------------------------------- body decoder (row R9, csrc/upconv_wnub.cu) */

/* replaces blocks.UpConvBlockDeep.forward (ca_code/nn/blocks.py:382-434): UpsamplingBilinear2d (align_corners=True,
 * x2), the weight-normalised grouped conv_resize 1x1 (tied bias), conv1 / conv2 3x3 "same" (la.Conv2dUB, untied bias
 * [C,2Hi,2Wi], layers.py:276-327) and both LeakyReLUs, in two kernels; u and the skip are never written.
 * x [B,Cin,Hi,Wi]; v1 [Cin,Cin/G,3,3], v2 [Cout,Cin/G,3,3], vr [Cout,Cin/G]; s1 / s2 / sr = weight_g / ||weight_v||_F
 * per output channel; b1 [Cin,H,W], b2 [Cout,H,W], br [Cout].  h1 [B,Cin,H,W] (conv1's activation, kept for the
 * backward), out [B,Cout,H,W]; mask [B,Cout,H,W] uint8 = conv2's pre-activation > 0, or NULL when no backward follows. */
int gb_upconv_block_fwd(int B, int Cin, int Cout, int groups, int Hi, int Wi, const float* x, const float* v1,
                        const float* s1, const float* b1, const float* v2, const float* s2, const float* b2,
                        const float* vr, const float* sr, const float* br, float slope, float* h1, float* out,
                        unsigned char* mask, void* stream);
/* backward of the above (replaces the autograd graph of the same lines).  Scratch gz2 [B,Cout,H,W], gz1 and gu
 * [B,Cin,H,W]; gb1 [Cin,H,W], gb2 [Cout,H,W], gbr [Cout] and the effective-weight gradients at unit scale gw1, gw2, gwr
 * are all WRITTEN.  gx [B,Cin,Hi,Wi] or NULL is a gather over the upsample's footprint.  Every sum runs in a fixed order
 * (no float atomics), so the gradients are bitwise repeatable.
 * `workspace`: gb_upconv_block_bwd_workspace_bytes(B, Cin, Cout, groups, Hi, Wi) bytes. */
size_t gb_upconv_block_bwd_workspace_bytes(int B, int Cin, int Cout, int groups, int Hi, int Wi);
int gb_upconv_block_bwd(int B, int Cin, int Cout, int groups, int Hi, int Wi, const float* x, const float* v1,
                        const float* s1, const float* v2, const float* s2, const float* vr, const float* sr,
                        const float* h1, const unsigned char* mask, const float* gout, float slope, float* gz2,
                        float* gz1, float* gu, float* gb1, float* gb2, float* gbr, float* gw1, float* gw2, float* gwr,
                        float* gx, void* workspace, void* stream);

/* replaces impaint_batch / resample_tex (ca_code/utils/seams.py:14-41: index_put of src texels into dst texels,
 * (1-w) tex + w grid_sample(tex, 2(uv-0.5)) with align_corners=False and border padding) and sample_uv
 * (ca_code/utils/geom.py:273-304: grid_sample at vt with align_corners=True, zeros padding, then the mean over the
 * v2uv columns), forward and backward, as one fixed-order gather per output row:
 *   out[b, c, r] = sum_{e in [row_ptr[r], row_ptr[r+1])} coef[e] in[b, c, col[e]]
 * with element strides per tensor (in_bs / in_cs / in_rs per item / channel / row).  The backward is the same call on
 * the transposed table, built once per set of seam buffers, so both directions are deterministic. */
int gb_sparse_rows_apply(int B, int C, int n_rows, const int* row_ptr, const int* col, const float* coef,
                         const float* in, long long in_bs, long long in_cs, long long in_rs, float* out,
                         long long out_bs, long long out_cs, long long out_rs, void* stream);

/* replaces the 2048^2 part of mesh_vae.AutoEncoder.forward_tex (ca_code/models/mesh_vae.py:211-222: bilinear x2
 * upsample with align_corners=False, `+ upscale_net(x)`, `* tex_std + tex_mean`, `* shadow_map`) together with the
 * end of UpscaleNet.forward (mesh_vae.py:670-678: the 4 -> 12 1x1 out_block with untied bias, then PixelShuffle(2)):
 *   out[b,c,y,x] = ((U(t1)[b,c,y,x] + z[b, 4c + 2(y%2) + x%2, y/2, x/2]) * tex_std + tex_mean[c,y,x]) * s3[b,y,x],
 *   z[b,o,i,j] = scale[o] * sum_k v[o,k] h[b,k,i,j] + bias[o,i,j]
 * t1 [B,3,H,W], h [B,4,H,W], v [12,4] (out_block.weight_v), scale [12] = weight_g / ||weight_v||_F, bias [12,H,W],
 * tex_mean [1,3,2H,2W], s3 [B,1,2H,2W], out [B,3,2H,2W].  Neither z, the upsampled map nor the pre-shadow texture is
 * written. */
int gb_body_tex_compose_fwd(int B, int H, int W, const float* t1, const float* h, const float* v, const float* scale,
                            const float* bias, float tex_std, const float* tex_mean, const float* s3, float* out,
                            void* stream);
/* backward of the above; recomputes the pre-shadow texture from t1, h and the weights.  g_t1 [B,3,H,W] (a gather over
 * the upsample's footprint, no atomics), g_h [B,4,H,W], g_bias [12,H,W] (batch sum) and g_s3 [B,1,2H,2W] written;
 * g_w [12,4] ACCUMULATED (caller zeroes it) = gradient of the effective weight at unit scale, summed in a fixed order
 * through `workspace` (gb_body_tex_compose_workspace_bytes(H, W) bytes), so repeated calls are bitwise equal. */
size_t gb_body_tex_compose_workspace_bytes(int H, int W);
int gb_body_tex_compose_bwd(int B, int H, int W, const float* t1, const float* h, const float* v, const float* scale,
                            const float* bias, float tex_std, const float* tex_mean, const float* s3,
                            const float* g_out, float* g_t1, float* g_h, float* g_bias, float* g_w, float* g_s3,
                            float* workspace, void* stream);

/* ---------------------------------------------------------------- body render (csrc/mesh_raster.cu)
 * Conventions (DESIGN.md R9'', PARITY UNPINNED: drtk is outside the reference tree): pixel (x, y) samples the screen
 * point (x + 0.5, y + 0.5); a face is drawn only if its three vertices have z > 0 (no near clipping, no backface
 * culling) and its screen area is non-zero; the inside test is inclusive (every screen-space barycentric
 * lambda_k >= 0) for either winding; perspective-correct barycentrics b_k = (lambda_k / z_k) / sum_j lambda_j / z_j
 * and depth = 1 / sum_j lambda_j / z_j. */

/* replaces drtk.rasterize(v_pix, vi, h, w) (ca_code/utils/render_drtk.py:47).  v_pix [B,V,3] (x, y in pixels, z =
 * camera depth), vi [F,3] int32, index_img [B,H,W] int32 out (-1 = background).  Each pixel keeps the face with the
 * smallest key (float_bits(depth) << 32) | face_id: the smaller depth, then the smaller face id, in any launch order.
 * Faces with a pixel box over 256 samples are rasterised one CTA per face.  Bit-exact with oracle/mesh_oracle.c.
 * `workspace`: gb_mesh_raster_workspace_bytes(B, F, H, W) bytes. */
size_t gb_mesh_raster_workspace_bytes(int B, int F, int H, int W);
int gb_mesh_raster(int B, int V, int F, int H, int W, const float* v_pix, const int32_t* vi, int32_t* index_img,
                   void* workspace, void* stream);
/* replaces drtk.render + drtk.interpolate of (2 vt - 1) + F.grid_sample(tex, vt_img, bilinear, align_corners=False,
 * zero padding) * mask (render_drtk.py:48-63), one thread per pixel.  vti [F,3] int32, vt [Vt,2], tex [B,C,Ht,Wt];
 * outputs depth_img [B,H,W] (0 on the background), bary_img [B,3,H,W], vt_img [B,2,H,W], mask [B,1,H,W] and render
 * [B,C,H,W], each written once. */
int gb_mesh_render_fwd(int B, int V, int F, int H, int W, int C, int Ht, int Wt, const float* v_pix, const int32_t* vi,
                       const int32_t* vti, const float* vt, const float* tex, const int32_t* index_img,
                       float* depth_img, float* bary_img, float* vt_img, float* mask, float* render, void* stream);
/* replaces the autograd graph of render_drtk.py:45-73 from `render` to v_pix and tex, including
 * drtk.edge_grad_estimator when edge_grad != 0 (the project's estimator, DESIGN.md R9'').  g_v_pix [B,V,3] and g_tex
 * [B,C,Ht,Wt] are written, bitwise repeatable (no float atomics): per-pixel records stably sorted by face and by
 * texel, fixed-order sums per face and per texel, and a vertex gather over the CSR list inc_ptr [V+1] / inc [3F]
 * (entries 3 f + corner, grouped by vertex, ascending within a vertex) that the caller builds once per vi.
 * `workspace`: gb_mesh_render_bwd_workspace_bytes(B, F, H, W, Ht, Wt) bytes. */
size_t gb_mesh_render_bwd_workspace_bytes(int B, int F, int H, int W, int Ht, int Wt);
int gb_mesh_render_bwd(int B, int V, int F, int H, int W, int C, int Ht, int Wt, const float* v_pix, const int32_t* vi,
                       const int32_t* vti, const float* vt, const float* tex, const int32_t* index_img,
                       const float* vt_img, const float* render, const float* g_render, int edge_grad,
                       const int32_t* inc_ptr, const int32_t* inc, float* g_v_pix, float* g_tex, void* workspace,
                       void* stream);

/* ---------------------------------------------------------------- body encoders (row R9''', csrc/downconv_wnub.cu) */

/* replaces blocks.ConvDownBlock.forward (ca_code/nn/blocks.py:327-379): conv1 3x3 stride 1 and conv2 3x3 stride 2
 * pad 1 (la.Conv2dUB, untied biases [Cin,H,W] and [Cout,H/2,W/2]), both LeakyReLUs and the weight-normalised grouped
 * conv_resize 1x1 stride 2 (tied bias), in two kernels; the skip is never written.  H and W (the input size) are even.
 * x is read through element strides x_bs (item), x_cs (channel), x_rs (row), unit along a row.  With cond_mask == NULL
 * x is [B,Cin,H,W] (Hs = H, Ws = W).  With cond_mask [H,W] uint8 the block's input is
 *   cond_scale * bilinear(x [B,Cin,Hs,Ws] -> H x W, align_corners = False) * cond_mask
 * evaluated while tiles are staged (replaces mesh_vae.py:394-399, and the crop of mesh_vae.py:434 through the strides).
 * v1 [Cin,Cin/G,3,3], v2 [Cout,Cin/G,3,3], vr [Cout,Cin/G]; s1 / s2 / sr = weight_g / ||weight_v||_F per output
 * channel; b1 [Cin,H,W], b2 [Cout,H/2,W/2], br [Cout].  h1 [B,Cin,H,W] (conv1's activation, kept for the backward),
 * out [B,Cout,H/2,W/2]; mask [B,Cout,H/2,W/2] uint8 = conv2's pre-activation > 0, or NULL when no backward follows. */
int gb_downconv_block_fwd(int B, int Cin, int Cout, int groups, int H, int W, const float* x, long long x_bs,
                          long long x_cs, int x_rs, int Hs, int Ws, const unsigned char* cond_mask, float cond_scale,
                          const float* v1, const float* s1, const float* b1, const float* v2, const float* s2,
                          const float* b2, const float* vr, const float* sr, const float* br, float slope, float* h1,
                          float* out, unsigned char* mask, void* stream);
/* backward of the above (replaces the autograd graph of the same lines).  Scratch gz2 [B,Cout,H/2,W/2] and gz1
 * [B,Cin,H,W]; gb1 [Cin,H,W], gb2 [Cout,H/2,W/2], gbr [Cout] and the effective-weight gradients at unit scale gw1, gw2,
 * gwr are all WRITTEN.  gx [B,Cin,H,W] or NULL (it must be NULL with cond_mask: the resize has no backward).  Every sum
 * runs in a fixed order (no float atomics), so the gradients are bitwise repeatable.
 * `workspace`: gb_downconv_block_bwd_workspace_bytes(B, Cin, Cout, groups, H, W) bytes. */
size_t gb_downconv_block_bwd_workspace_bytes(int B, int Cin, int Cout, int groups, int H, int W);
int gb_downconv_block_bwd(int B, int Cin, int Cout, int groups, int H, int W, const float* x, long long x_bs,
                          long long x_cs, int x_rs, int Hs, int Ws, const unsigned char* cond_mask, float cond_scale,
                          const float* v1, const float* s1, const float* v2, const float* s2, const float* vr,
                          const float* sr, const float* h1, const unsigned char* mask, const float* gout, float slope,
                          float* gz2, float* gz1, float* gb1, float* gb2, float* gbr, float* gw1, float* gw2,
                          float* gwr, float* gx, void* workspace, void* stream);

/* ---------------------------------------------------------------- body frame (row R9'''', csrc/body_frame.cu) */

/* replaces geom.depth_discontuity_mask (ca_code/utils/geom.py:768-794) with its pool_ksize 3: Sobel x / y of depth
 * [B,1,H,W] with zero padding, sqrt(gx^2 + gy^2) > threshold (evaluated in double), then the 3x3 stride-1 avg_pool > 0,
 * i.e. any such pixel among the neighbours inside the image.  mask [B,1,H,W] uint8 (torch.bool) is written once.
 * Forward only: the reference runs it under no_grad on a detached depth (mesh_vae.py:320-322). */
int gb_depth_disc_mask(int B, int H, int W, const float* depth, float threshold, unsigned char* mask, void* stream);
/* replaces rgb + CameraPixelBias(idx) (ca_code/models/mesh_vae.py:51-69 and :335-339):
 *   out[b,c] = rgb[b,c] + bilinear(bias[idx[b]] [Hb,Wb] -> H x W, align_corners = False)
 * rgb / out [B,C,H,W], bias [n_cams,1,Hb,Wb] (the reference's parameter is [n_cams,1,W/ds,H/ds]: Hb = W/ds is stretched
 * over H), idx [B] int64 (an index outside [0, n_cams) adds nothing).  out may not alias rgb. */
int gb_pixel_bias_fwd(int B, int C, int H, int W, int n_cams, int Hb, int Wb, const float* rgb, const float* bias,
                      const long long* idx, float* out, void* stream);
/* the bias gradient of the above: g_bias [n_cams,1,Hb,Wb] is WRITTEN, one thread per camera and texel, summing its
 * upsample footprint over the C channels and over the items b with idx[b] == camera in batch order (no float atomics:
 * the same bits on every call).  The rgb gradient is g_out itself. */
int gb_pixel_bias_bwd(int B, int C, int H, int W, int n_cams, int Hb, int Wb, const long long* idx, const float* g_out,
                      float* g_bias, void* stream);

/* ---------------------------------------------------------------- drivable body (row R10, csrc/body_drive.cu) */

/* replaces the last ConvTranspose2dWNUB of FaceDecoderFrontal.texmod and face.py:80-82 (ca_code/nn/face.py:58,78-82):
 *   tex_raw = ConvTranspose2d(x, weight_v, k = 4, s = 2, p = 1) * scale[co] + bias      (scale = g / ||weight_v||_F)
 *   tex     = 255 * (tex_raw + face_bias + 0.5)
 * x [B,Cin,Hi,Wi] with Cin <= 32, weight_v [Cin,Cout,4,4] with Cout <= 4, scale [Cout], bias and face_bias
 * [Cout,2Hi,2Wi]; tex_raw and tex [B,Cout,2Hi,2Wi] are each written once.  Forward only (the frame runs the face
 * decoder under no_grad, mesh_vae_drivable.py:276-277). */
int gb_face_tex_tail_fwd(int B, int Cin, int Cout, int Hi, int Wi, const float* x, const float* weight_v,
                         const float* scale, const float* bias, const float* face_bias, float* tex_raw, float* tex,
                         void* stream);
/* replaces FaceEncoder's conditioning (ca_code/models/mesh_vae_drivable.py:721-724):
 *   out[b,c] = (bilinear(x[b,c] [Hs,Ws] -> H x W, align_corners = False) / 255 - 0.5) * mask
 * with torch's fp32 half-pixel source index, for any source size; x [B,C,Hs,Ws], mask [H,W], out [B,C,H,W].
 * Forward only. */
int gb_face_tex_cond_fwd(int B, int C, int Hs, int Ws, int H, int W, const float* x, const float* mask, float* out,
                         void* stream);
/* replaces PoseToShadow's sigmoid + resize (ca_code/nn/shadow.py:466-470):
 *   out[n] = bilinear(sigmoid(x[n] + beta) [h,w] -> H x W, align_corners = False)
 * x [N,h,w] (N = B * C planes), out [N,H,W]; torch's fp32 half-pixel index, the sigmoid evaluated at the taps. */
int gb_pose_shadow_fwd(int N, int h, int w, int H, int W, const float* x, float beta, float* out, void* stream);
/* the x gradient of the above: g_x [N,h,w] is WRITTEN, one thread per low-resolution texel, gathering its upsample
 * footprint of g_out [N,H,W] in row-major order and multiplying by sigmoid' (no float atomics: the same bits on every
 * call). */
int gb_pose_shadow_bwd(int N, int h, int w, int H, int W, const float* x, float beta, const float* g_out, float* g_x,
                       void* stream);

/* ---------------------------------------------------------------- head frame (row R11, csrc/head_frame.cu) */

/* replaces the head-relative light work of rgca.AutoEncoder.forward (ca_code/models/rgca.py:175-193), one CTA per
 * batch item:
 *   headrel_Rt [B,3,4]         = Rt @ [head_pose; 0 0 0 1]
 *   headrel_campos [B,3]       = (campos - t) @ R                          (R | t = head_pose [B,3,4])
 *   headrel_light_pos [B,L,3]  = (light_pos - t) @ R
 *   headrel_light_sh [B,3,81]  = sum over all L lights of dir2sh(8, normalize(headrel_light_pos)) * intensity
 *   lightrot_out [B,3,3]       = lightrot @ R                              (both NULL when there is no lightrot)
 * light_intensity [B,L,C] with C = 1 (used for all three channels, rgca.py:175) or 3.  The direction follows
 * F.normalize's max(|v|, 1e-12); the basis is sh.dir2sh's.  Double arithmetic from the fp32 inputs; the sum over L
 * runs in index order with no atomics, so two calls give the same bits.  Forward only (none of the inputs carries a
 * gradient in the reference's use). */
int gb_head_lights_fwd(int B, int L, int C, const float* head_pose, const float* campos, const float* Rt,
                       const float* light_pos, const float* light_intensity, const float* lightrot, float* headrel_Rt,
                       float* headrel_campos, float* headrel_light_pos, float* headrel_light_sh, float* lightrot_out,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GOLIATH_B200_H_ */
