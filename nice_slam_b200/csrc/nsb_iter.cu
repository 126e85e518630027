// nsb_iter.cu -- one optimisation iteration enqueued by a single C call:
//   batch depth maxima -> render forward -> loss seeds -> render backward
// (Tracker.optimize_cam_in_batch, src/Tracker.py:106-125; one joint_iter of Mapper.optimize_map, src/Mapper.py:482-503).
#include <cstring>
#include "nsb_common.cuh"

using namespace nsb;

// workspace = [fused-seeds counter (16 B) | tracking-seeds scratch | packed weight-gradient images | tile-kernel workspace = the rest].
// Only the first 16 bytes and the END of the buffer (ray completion counters, nsb_render.cu) hold state that must stay zero between calls,
// so one buffer sized for a capacity serves batches of varying size.
static size_t backward_offset(int n_rays) { return 16 + align16(nsb_tracking_seeds_workspace(n_rays)); }
static size_t split_offset(int n_rays) { return backward_offset(n_rays) + align16(nsb_backward_workspace_bytes()); }
extern "C" size_t nsb_iteration_workspace_bytes(int n_rays) {
  return split_offset(n_rays) + align16(nsb_split_workspace_bytes(n_rays, NSB_MAX_SAMPLES));
}
struct IterWs { int* seeds_counter; void* seeds_scratch; void* backward; void* split; size_t split_bytes; };
static IterWs carve(const nsb_iteration_buffers* b, int n_rays) {
  char* w = static_cast<char*>(b->workspace);
  return {reinterpret_cast<int*>(w), w + 16, w + backward_offset(n_rays), w + split_offset(n_rays), b->workspace_bytes - split_offset(n_rays)};
}

static int check_buffers(const nsb_render_inputs* in, const nsb_iteration_buffers* b, const nsb_backward_args* g) {
  if (!in || !b || !g) { set_error("iteration: NULL argument"); return NSB_ERR_ARG; }
  if (!b->depth || !b->var || !b->rgb || !b->z_vals || !b->raw || !b->g_depth || !b->g_rgb || !b->loss || !b->depth_max || !b->workspace) {
    set_error("iteration: incomplete nsb_iteration_buffers"); return NSB_ERR_ARG; }
  if (b->workspace_bytes < nsb_iteration_workspace_bytes(in->n_rays)) {
    int det = 0; nsb_get_option("deterministic", &det);
    set_error(det ? "iteration: workspace smaller than nsb_iteration_workspace_bytes(%d) with option deterministic on (size it after setting the option)"
                  : "iteration: workspace too small", in->n_rays);
    return NSB_ERR_ARG;
  }
  return NSB_OK;
}

static int forward_part(const nsb_render_inputs* in, const nsb_iteration_buffers* b, const IterWs& ws, nsb_render_inputs* in2, const FusedSeeds* fs,
                        void* stream, bool keep_depth_max = false) {
  *in2 = *in;
  if (!(keep_depth_max && in->depth_max != nullptr)) {             // else the caller supplies the batch depth maxima (sharded batch: maxima of the FULL batch)
    in2->depth_max = nullptr;
    if (in->gt_depth && in->gt_depth_batch == nullptr && in->n_rays > NSB_INLINE_MAX_RAYS) {        // small batches: the render kernel reduces gt_depth itself
      const int rc = nsb_batch_max_depth(in->gt_depth, in->n_rays, b->depth_max, stream); if (rc) return rc;
      in2->depth_max = b->depth_max;
    }
  }
  nsb_forward_outputs fo = {b->depth, b->var, b->rgb, b->z_vals, b->raw, nullptr, b->masks, ws.split, ws.split_bytes, b->acts, b->acts_levels};
  return render_forward_fused(in2, &fo, fs, stream);
}

// loss seeds computed by the forward's last CTA into the iteration buffers: kind 1 = tracking (with the residual scratch of the median),
// 2 = mapping; px: the exchange of a ray-sharded batch, or NULL
static FusedSeeds fused_seeds(const nsb_iteration_buffers* b, const IterWs& ws, int kind, const void* gt_rgb, const float* gt_depth_loss, double w_color,
                              int handle_dynamic, int use_color, const PeerX* px) {
  FusedSeeds fs; memset(&fs, 0, sizeof(fs));
  fs.kind = kind; fs.gt_rgb = gt_rgb; fs.gt_depth_loss = gt_depth_loss; fs.w_color = w_color; fs.handle_dynamic = handle_dynamic; fs.use_color = use_color;
  fs.g_depth = b->g_depth; fs.g_rgb = b->g_rgb; fs.loss = b->loss; fs.counter = ws.seeds_counter;
  if (kind == 1) fs.res = static_cast<double*>(ws.seeds_scratch);
  if (px != nullptr) fs.px = *px;
  return fs;
}

static int backward_part(const nsb_render_inputs* in2, const nsb_iteration_buffers* b, const IterWs& ws, const nsb_backward_args* g, void* stream,
                         const PeerTail* tail = nullptr, bool after_forward = false) {
  nsb_backward_args bw = *g;
  bw.z_vals = b->z_vals; bw.raw = b->raw; bw.g_depth = b->g_depth; bw.g_var = nullptr; bw.g_rgb = b->g_rgb; bw.masks = b->masks; bw.acts = b->acts; bw.acts_levels = b->acts_levels;
  bw.workspace = ws.backward; bw.split_workspace = ws.split; bw.split_workspace_bytes = ws.split_bytes;
  if (b->event_bwd_begin) cudaEventRecord((cudaEvent_t)b->event_bwd_begin, (cudaStream_t)stream);
  const int rc = render_backward_tail(in2, &bw, tail, stream, after_forward && !b->event_bwd_begin);
  if (b->event_bwd_end) cudaEventRecord((cudaEvent_t)b->event_bwd_end, (cudaStream_t)stream);
  return rc;
}

extern "C" int nsb_tracking_iteration(const nsb_render_inputs* in, const nsb_iteration_buffers* buf, const double* gt_rgb,
                                      double w_color, int handle_dynamic, int use_color, const nsb_backward_args* grads, void* stream) {
  int rc = check_buffers(in, buf, grads); if (rc) return rc;
  if (!in->gt_depth) { set_error("tracking iteration needs gt_depth"); return NSB_ERR_ARG; }
  nsb_render_inputs in2;
  // small batches: the last CTA of the forward launch computes the loss seeds itself (no separate single-CTA launch)
  const bool fuse = in->n_rays > 0 && in->n_rays <= 512;          // (the median by direct rank counting, nsb_seeds.cuh)
  if (fuse && use_color && !gt_rgb) { set_error("tracking iteration: use_color without gt_rgb"); return NSB_ERR_ARG; }
  const IterWs ws = carve(buf, in->n_rays);
  const FusedSeeds fs = fused_seeds(buf, ws, 1, gt_rgb, nullptr, w_color, handle_dynamic, use_color, nullptr);
  if ((rc = forward_part(in, buf, ws, &in2, fuse ? &fs : nullptr, stream))) return rc;
  if (!fuse && (rc = nsb_tracking_seeds(buf->depth, buf->var, buf->rgb, in->gt_depth, gt_rgb, in->n_rays, w_color, handle_dynamic, use_color,
                                        nullptr, 0, buf->g_depth, buf->g_rgb, buf->loss, ws.seeds_scratch, nsb_tracking_seeds_workspace(in->n_rays), stream))) return rc;
  return backward_part(&in2, buf, ws, grads, stream, nullptr, fuse);
}

// Ray-sharded tracking iteration in TWO launches per rank: the forward exchanges the depth maxima (every CTA) and the residual pool of the
// median (last CTA, which then computes the loss seeds); the backward's last CTA sums [loss | d c2w] over the ranks.
extern "C" int nsb_tracking_iteration_peers(const nsb_render_inputs* in, const nsb_iteration_buffers* buf, const double* gt_rgb,
                                            double w_color, int handle_dynamic, int use_color, const nsb_backward_args* grads,
                                            const nsb_peers* peers, double* loss_and_d_c2w, void* stream) {
  int rc = check_buffers(in, buf, grads); if (rc) return rc;
  if (!in->gt_depth || !loss_and_d_c2w) { set_error("sharded tracking iteration needs gt_depth and an output for [loss | d c2w]"); return NSB_ERR_ARG; }
  if (in->n_rays < 1 || in->n_rays > 512) { set_error("sharded tracking iteration: 1..512 rays per rank (got %d)", in->n_rays); return NSB_ERR_UNSUPPORTED; }
  if (!grads->pose_dirs || !grads->d_c2w || !grads->pose_counter) { set_error("sharded tracking iteration needs pose_dirs / d_c2w / pose_counter"); return NSB_ERR_ARG; }
  if (use_color && !gt_rgb) { set_error("tracking iteration: use_color without gt_rgb"); return NSB_ERR_ARG; }
  PeerX px;
  if ((rc = make_peerx(peers, &px))) return rc;
  if (in->n_rays > px.max_n) { set_error("sharded tracking iteration: %d rays exceed the exchange buffers' capacity %d", in->n_rays, px.max_n); return NSB_ERR_ARG; }
  const IterWs ws = carve(buf, in->n_rays);
  const FusedSeeds fs = fused_seeds(buf, ws, 1, gt_rgb, nullptr, w_color, handle_dynamic, use_color, &px);
  nsb_render_inputs in2;
  if ((rc = forward_part(in, buf, ws, &in2, &fs, stream, true))) return rc;      // in->depth_max given: no depth-max exchange inside the forward
  PeerTail tail; tail.px = px; tail.loss = buf->loss; tail.out13 = loss_and_d_c2w;
  return backward_part(&in2, buf, ws, grads, stream, &tail, true);
}

extern "C" int nsb_mapping_iteration(const nsb_render_inputs* in, const nsb_iteration_buffers* buf, const float* gt_depth_loss,
                                     const float* gt_rgb, double w_color, const nsb_backward_args* grads, void* stream) {
  int rc = check_buffers(in, buf, grads); if (rc) return rc;
  const float* gtl = gt_depth_loss ? gt_depth_loss : in->gt_depth;
  if (!gtl) { set_error("mapping iteration needs a depth to supervise with"); return NSB_ERR_ARG; }
  nsb_render_inputs in2;
  const int use_color = in->stage == NSB_STAGE_COLOR;                      // Mapper.py:490
  const bool fuse = in->n_rays > 0 && in->n_rays <= NSB_INLINE_MAX_RAYS;
  if (fuse && use_color && !gt_rgb) { set_error("mapping iteration: colour stage without gt_rgb"); return NSB_ERR_ARG; }
  const IterWs ws = carve(buf, in->n_rays);
  const FusedSeeds fs = fused_seeds(buf, ws, 2, gt_rgb, gtl, w_color, 0, use_color, nullptr);
  if ((rc = forward_part(in, buf, ws, &in2, fuse ? &fs : nullptr, stream))) return rc;
  if (!fuse && (rc = nsb_mapping_seeds(buf->depth, buf->rgb, gtl, gt_rgb, in->n_rays, w_color, use_color, buf->g_depth, buf->g_rgb, buf->loss, stream))) return rc;
  return backward_part(&in2, buf, ws, grads, stream, nullptr, fuse);
}
