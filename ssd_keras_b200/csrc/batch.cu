// Batch assembly for the ground-truth encoder: the box half of the reference's augmentation chain on the device, and the
// packing of the surviving boxes into the encoder's ragged (sum G_i x 5, offsets) format.
// Reference: the label arithmetic of CropPad (data_generator/object_detection_2d_patch_sampling_ops.py:258-330, used by
// SSDExpand / SSDRandomCrop through RandomPatch), Flip (object_detection_2d_geometric_ops.py:171-195), Resize (:61-100),
// BoxFilter (object_detection_2d_image_boxes_validation_utils.py:120-200), and the degenerate-box handling + hand-off to the
// label encoder in DataGenerator.generate (object_detection_2d_data_generator.py:1095-1151).
// The random decisions of the chain (which patch, flip or not) are host-side control flow in the reference and stay with the
// caller: this file takes the decided parameters as a per-image list of box operations.
//   box_ops_kernel     one CTA per image: every box through the image's operation list in float64 (what NumPy computes on
//                      int / float64 label arrays; np.round = round-half-even = rint), a validity flag per box, ordered
//                      compaction of the survivors.
//   box_offsets_kernel one CTA: exclusive scan of the survivor counts -> row offsets, total and maximum.
//   box_pack_kernel    one CTA per image: rows to their final place.
// The image half of the same op lists (ssdk_assemble_images) is at the end of the file: ConvertTo3Channels
// (object_detection_2d_photometric_ops.py:88-108), the image arithmetic of CropPad (:266-313) and Flip, and uint8 cv2.resize
// (INTER_NEAREST / INTER_LINEAR) in one launch, restated in oracle/imageops.py.
//   image_assemble_kernel  one CTA per (output row, image): every output pixel is traced back through the resize to at most
//                          four canvas taps, and each tap through the composed crop / pad / flip map to a source pixel or to
//                          the background colour.  No intermediate image exists.
// The file is compiled with --fmad=false; the float64 resize coordinates also spell their roundings out (__dmul_rn / __dadd_rn).
#include "common.cuh"
#include <cmath>
#include <vector>

using namespace ssdk;

namespace {

constexpr int kBoxThreads = 128;

__global__ void __launch_bounds__(kBoxThreads) box_ops_kernel(const void* __restrict__ gt, int gt_f64, const int* __restrict__ offs, const ssdk_box_op* __restrict__ ops,
                                                              int max_ops, float* __restrict__ tmp, int* __restrict__ counts) {
  __shared__ int s_w[kBoxThreads / 32];
  __shared__ int s_base;
  const int b = blockIdx.x;
  const int g0 = offs[b], G = offs[b + 1] - g0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  for (int base = 0; base < G; base += kBoxThreads) {
    const int g = base + threadIdx.x;
    bool valid = g < G;
    double cls = 0, x0 = 0, y0 = 0, x1 = 0, y1 = 0;
    if (valid) {
      if (gt_f64) { const double* r = reinterpret_cast<const double*>(gt) + (size_t)(g0 + g) * 5; cls = r[0]; x0 = r[1]; y0 = r[2]; x1 = r[3]; y1 = r[4]; }
      else { const float* r = reinterpret_cast<const float*>(gt) + (size_t)(g0 + g) * 5; cls = r[0]; x0 = r[1]; y0 = r[2]; x1 = r[3]; y1 = r[4]; }
      for (int i = 0; i < max_ops; ++i) {
        const ssdk_box_op op = ops[(size_t)b * max_ops + i];
        if (op.op == SSDK_BOXOP_END) break;
        if (op.op == SSDK_BOXOP_CROP_PAD) {
          // labels -= patch origin; BoxFilter 'center_point' against the patch; clip to the patch (CropPad.__call__)
          y0 -= op.a0; y1 -= op.a0; x0 -= op.a1; x1 -= op.a1;
          if (op.flags & 1) {
            const double cy = (y0 + y1) / 2, cx = (x0 + x1) / 2;
            valid = valid && (cy >= 0.0) && (cy <= op.a2 - 1) && (cx >= 0.0) && (cx <= op.a3 - 1);
          }
          if (op.flags & 2) {
            y0 = fmin(fmax(y0, 0.0), op.a2 - 1); y1 = fmin(fmax(y1, 0.0), op.a2 - 1);
            x0 = fmin(fmax(x0, 0.0), op.a3 - 1); x1 = fmin(fmax(x1, 0.0), op.a3 - 1);
          }
        } else if (op.op == SSDK_BOXOP_FLIP_H) {             // labels[:, [xmin, xmax]] = img_width - labels[:, [xmax, xmin]]
          const double nx0 = op.a0 - x1, nx1 = op.a0 - x0; x0 = nx0; x1 = nx1;
        } else if (op.op == SSDK_BOXOP_FLIP_V) {
          const double ny0 = op.a0 - y1, ny1 = op.a0 - y0; y0 = ny0; y1 = ny1;
        } else if (op.op == SSDK_BOXOP_RESIZE) {             // np.round(labels * (out / in), decimals=0)
          const double sy = op.a2 / op.a0, sx = op.a3 / op.a1;
          y0 = rint(y0 * sy); y1 = rint(y1 * sy); x0 = rint(x0 * sx); x1 = rint(x1 * sx);
          if (op.flags & 1) valid = valid && (x1 > x0) && (y1 > y0);
        } else if (op.op == SSDK_BOXOP_FILTER) {             // BoxFilter: degenerate and / or minimum area
          if (op.flags & 1) valid = valid && (x1 > x0) && (y1 > y0);
          if (op.flags & 2) valid = valid && ((x1 - x0) * (y1 - y0) >= op.a0);
        }
      }
    }
    // ordered compaction (box order is kept, like labels[requirements_met])
    const unsigned m = __ballot_sync(0xffffffffu, valid);
    if (lane == 0) s_w[warp] = __popc(m);
    __syncthreads();
    int before = s_base, total = 0;
    for (int w = 0; w < kBoxThreads / 32; ++w) { if (w < warp) before += s_w[w]; total += s_w[w]; }
    if (valid) {
      float* o = tmp + (size_t)(g0 + before + __popc(m & ((1u << lane) - 1))) * 5;
      o[0] = (float)cls; o[1] = (float)x0; o[2] = (float)y0; o[3] = (float)x1; o[4] = (float)y1;
    }
    __syncthreads();
    if (threadIdx.x == 0) s_base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[b] = s_base;
}

__global__ void __launch_bounds__(1024) box_offsets_kernel(const int* __restrict__ counts, int B, int* __restrict__ offs_out, int* __restrict__ stats) {
  __shared__ int s_sum[1024];
  __shared__ int s_max[1024];
  const int t = threadIdx.x;
  const int per = (B + 1023) / 1024;
  const int lo = t * per, hi = min(B, lo + per);
  int sum = 0, mx = 0;
  for (int i = lo; i < hi; ++i) { sum += counts[i]; mx = max(mx, counts[i]); }
  s_sum[t] = sum; s_max[t] = mx;
  __syncthreads();
  int base = 0;
  for (int i = 0; i < t; ++i) base += s_sum[i];
  for (int i = lo; i < hi; ++i) { offs_out[i] = base; base += counts[i]; }
  if (t == 1023) {
    int m = 0;
    for (int i = 0; i < 1024; ++i) m = max(m, s_max[i]);
    offs_out[B] = base;
    if (stats) { stats[0] = base; stats[1] = m; }
  }
}

__global__ void __launch_bounds__(kBoxThreads) box_pack_kernel(const float* __restrict__ tmp, const int* __restrict__ offs_in, const int* __restrict__ offs_out,
                                                               float* __restrict__ out) {
  const int b = blockIdx.x;
  const int n = (offs_out[b + 1] - offs_out[b]) * 5;
  const float* src = tmp + (size_t)offs_in[b] * 5;
  float* dst = out + (size_t)offs_out[b] * 5;
  for (int i = threadIdx.x; i < n; i += kBoxThreads) dst[i] = src[i];
}

}  // namespace

extern "C" int ssdk_assemble_batch(ssdk_ctx* ctx, const void* gt_in_dev, int gt_in_f64, const int* offsets_in_dev, int B, int total_in,
                                   const ssdk_box_op* ops_dev, int max_ops, float* gt_out_dev, int* offsets_out_dev, int* out_stats_dev,
                                   void* stream_) {
  SSDK_REQUIRE(ctx && offsets_in_dev && gt_out_dev && offsets_out_dev && B > 0 && total_in >= 0, "ssdk_assemble_batch: bad argument");
  SSDK_REQUIRE(total_in == 0 || gt_in_dev, "ssdk_assemble_batch: gt_in_dev is NULL");
  SSDK_REQUIRE(max_ops == 0 || ops_dev, "ssdk_assemble_batch: ops_dev is NULL");
  cudaStream_t stream = (cudaStream_t)stream_;
  const size_t need = (size_t)(total_in > 0 ? total_in : 1) * 5 * sizeof(float) + (size_t)B * sizeof(int) + 256;
  int rc = ctx->ws[3].ensure(need);
  if (rc) return rc;
  float* tmp = reinterpret_cast<float*>(ctx->ws[3].ptr);
  int* counts = reinterpret_cast<int*>(reinterpret_cast<unsigned char*>(ctx->ws[3].ptr) + (((size_t)(total_in > 0 ? total_in : 1) * 5 * sizeof(float) + 255) / 256 * 256));
  box_ops_kernel<<<B, kBoxThreads, 0, stream>>>(gt_in_dev, gt_in_f64, offsets_in_dev, ops_dev, max_ops, tmp, counts);
  SSDK_COUNT_LAUNCH(ctx);
  box_offsets_kernel<<<1, 1024, 0, stream>>>(counts, B, offsets_out_dev, out_stats_dev);
  SSDK_COUNT_LAUNCH(ctx);
  box_pack_kernel<<<B, kBoxThreads, 0, stream>>>(tmp, offsets_in_dev, offsets_out_dev, gt_out_dev);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// ------------------------------------------------------------------------------------------------
// Images
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int kImgThreads = 128;
enum { kImgCopy = 0, kImgNearest = 1, kImgLinear = 2, kImgArea2 = 3 };

// One image's op list, composed on the host.  Every crop, pad and flip before the resize is an integer translation and / or
// reflection per axis, so the canvas the resize reads is described by its size, one affine map to the source and the rectangle
// the source covers; canvas pixels outside that rectangle show the background colour.
struct ImgDesc {
  long long src_off;           // byte offset of the image in the packed source buffer
  int h, w, c;                 // source geometry (c = 1, 3 or 4)
  int ch, cw;                  // canvas size before the resize
  int oy, sy, ox, sx;          // source row = oy + sy * canvas row, source column = ox + sx * canvas column (sy, sx = +-1)
  int vy0, vy1, vx0, vx1;      // canvas rows [vy0, vy1) x columns [vx0, vx1) come from the source
  int bg;                      // background R | G << 8 | B << 16
  int mode;                    // kImgCopy / kImgNearest / kImgLinear / kImgArea2
  double scale_y, scale_x;     // cv2's 1 / (out / in), float64
};

__device__ __forceinline__ void canvas_px(const uint8_t* __restrict__ src, const ImgDesc& d, int r, int c, int v[3]) {
  if (r >= d.vy0 && r < d.vy1 && c >= d.vx0 && c < d.vx1) {
    const uint8_t* p = src + d.src_off + ((long long)(d.oy + d.sy * r) * d.w + (d.ox + d.sx * c)) * d.c;
    if (d.c == 1) { v[0] = v[1] = v[2] = p[0]; }              // gray -> RGB by replication, RGBA -> RGB drops alpha
    else { v[0] = p[0]; v[1] = p[1]; v[2] = p[2]; }
  } else {
    v[0] = d.bg & 255; v[1] = (d.bg >> 8) & 255; v[2] = (d.bg >> 16) & 255;
  }
}

// cv2's INTER_LINEAR coordinate: fx = (float)((d + 0.5) * scale - 0.5), s = floor(fx), fx -= s.
__device__ __forceinline__ void linear_coord(int dst, double scale, int& s, float& f) {
  const float fx = __double2float_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)dst, 0.5), scale), -0.5));
  s = (int)floorf(fx);
  f = __fsub_rn(fx, (float)s);
}
// saturate_cast<short>(w * 2048): round half to even; w is in [0, 1] so no saturation is needed.
__device__ __forceinline__ int coef11(float w) { return __float2int_rn(__fmul_rn(w, 2048.f)); }

__global__ void __launch_bounds__(kImgThreads) image_assemble_kernel(const uint8_t* __restrict__ src, const ImgDesc* __restrict__ descs,
                                                                     int out_h, int out_w, float* __restrict__ out) {
  const int b = blockIdx.y, dy = blockIdx.x;
  const ImgDesc d = descs[b];
  float* orow = out + ((size_t)b * out_h + dy) * (size_t)out_w * 3;
  // the row taps are shared by the whole CTA; rows keep their fraction at the borders and read the edge row twice (resizeGeneric_)
  int r0 = dy, r1 = dy, b0 = 2048, b1 = 0;
  if (d.mode == kImgNearest) {
    r0 = min((int)floor(__dmul_rn((double)dy, d.scale_y)), d.ch - 1);
  } else if (d.mode == kImgLinear) {
    int s; float f;
    linear_coord(dy, d.scale_y, s, f);
    r0 = min(max(s, 0), d.ch - 1); r1 = min(max(s + 1, 0), d.ch - 1);
    b0 = coef11(__fsub_rn(1.f, f)); b1 = coef11(f);
  } else if (d.mode == kImgArea2) {
    r0 = 2 * dy; r1 = 2 * dy + 1;
  }
  for (int dx = threadIdx.x; dx < out_w; dx += kImgThreads) {
    int v[3];
    if (d.mode == kImgCopy) {
      canvas_px(src, d, r0, dx, v);
    } else if (d.mode == kImgNearest) {
      canvas_px(src, d, r0, min((int)floor(__dmul_rn((double)dx, d.scale_x)), d.cw - 1), v);
    } else if (d.mode == kImgArea2) {                         // INTER_AREA's fast 2x path: rounded mean of a 2x2 block
      int p[3], q[3], r[3];
      canvas_px(src, d, r0, 2 * dx, v); canvas_px(src, d, r0, 2 * dx + 1, p);
      canvas_px(src, d, r1, 2 * dx, q); canvas_px(src, d, r1, 2 * dx + 1, r);
#pragma unroll
      for (int k = 0; k < 3; ++k) v[k] = (v[k] + p[k] + q[k] + r[k] + 2) >> 2;
    } else {
      // columns past either border take the edge pixel with weight 2048
      int s; float f;
      linear_coord(dx, d.scale_x, s, f);
      if (s < 0) { s = 0; f = 0.f; }
      if (s >= d.cw - 1) { s = d.cw - 1; f = 0.f; }
      const int c1 = min(s + 1, d.cw - 1);
      const int a0 = coef11(__fsub_rn(1.f, f)), a1 = coef11(f);
      int p01[3], p10[3], p11[3];
      canvas_px(src, d, r0, s, v); canvas_px(src, d, r0, c1, p01);
      canvas_px(src, d, r1, s, p10); canvas_px(src, d, r1, c1, p11);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int S0 = v[k] * a0 + p01[k] * a1, S1 = p10[k] * a0 + p11[k] * a1;      // horizontal pass, int
        const int t = (((b0 * (S0 >> 4)) >> 16) + ((b1 * (S1 >> 4)) >> 16) + 2) >> 2;  // cv2's vertical pass on 8-bit
        v[k] = min(max(t, 0), 255);
      }
    }
    orow[dx * 3 + 0] = (float)v[0]; orow[dx * 3 + 1] = (float)v[1]; orow[dx * 3 + 2] = (float)v[2];
  }
}

bool is_int(double a) { return a == std::floor(a) && std::fabs(a) <= (double)(1 << 24); }

// Compose image b's op list into its descriptor; every check the entry point documents.
int compose_image(int b, const long long* offs, const int* hwc, const ssdk_box_op* ops, int max_ops, int out_h, int out_w, ImgDesc* out) {
  const int h = hwc[3 * b], w = hwc[3 * b + 1], c = hwc[3 * b + 2];
  SSDK_REQUIRE(h > 0 && w > 0, "ssdk_assemble_images: image %d has size %dx%d", b, h, w);
  SSDK_REQUIRE(c == 1 || c == 3 || c == 4, "ssdk_assemble_images: image %d has %d channels (1, 3 or 4 are supported)", b, c);
  SSDK_REQUIRE(offs[b] >= 0 && offs[b + 1] - offs[b] == (long long)h * w * c,
               "ssdk_assemble_images: image %d: offsets %lld..%lld do not hold %dx%dx%d bytes", b, offs[b], offs[b + 1], h, w, c);
  long long ch = h, cw = w, oy = 0, ox = 0, vy0 = 0, vy1 = h, vx0 = 0, vx1 = w;
  int sy = 1, sx = 1, bg = 0, mode = kImgCopy;
  bool has_bg = false, resized = false;
  long long rh = 0, rw = 0;
  for (int i = 0; i < max_ops; ++i) {
    const ssdk_box_op& op = ops[(size_t)b * max_ops + i];
    if (op.op == SSDK_BOXOP_END) break;
    if (op.op == SSDK_BOXOP_FILTER) continue;                     // boxes only
    SSDK_REQUIRE(op.op >= SSDK_BOXOP_CROP_PAD && op.op <= SSDK_BOXOP_RESIZE, "ssdk_assemble_images: image %d, op %d: unknown op code %d", b, i, op.op);
    SSDK_REQUIRE(!resized, "ssdk_assemble_images: image %d, op %d: the RESIZE must be the last op that changes the image", b, i);
    if (op.op == SSDK_BOXOP_CROP_PAD) {
      SSDK_REQUIRE(is_int(op.a0) && is_int(op.a1) && is_int(op.a2) && is_int(op.a3) && op.a2 > 0 && op.a3 > 0,
                   "ssdk_assemble_images: image %d, op %d: CROP_PAD needs an integer patch of positive size", b, i);
      const long long py = (long long)op.a0, px = (long long)op.a1, ph = (long long)op.a2, pw = (long long)op.a3;
      SSDK_REQUIRE(!(py > ch || px > cw), "The given patch doesn't overlap with the input image. (image %d, op %d)", b, i);
      if (py < 0 || px < 0 || py + ph > ch || px + pw > cw) {     // the patch reaches past its input: it adds background
        const int col = (int)(((unsigned)op.flags >> 8) & 0xFFFFFFu);
        SSDK_REQUIRE(!has_bg || col == bg, "ssdk_assemble_images: image %d, op %d: two pads with different background colours in "
                     "one list are not supported", b, i);
        has_bg = true; bg = col;
      }
      oy += sy * py; ox += sx * px;
      vy0 = std::max(vy0 - py, 0LL); vy1 = std::min(vy1 - py, ph);
      vx0 = std::max(vx0 - px, 0LL); vx1 = std::min(vx1 - px, pw);
      if (vy1 <= vy0 || vx1 <= vx0) vy0 = vy1 = vx0 = vx1 = 0;      // nothing of the source is left
      ch = ph; cw = pw;
    } else if (op.op == SSDK_BOXOP_FLIP_H) {
      SSDK_REQUIRE(op.a0 == (double)cw, "ssdk_assemble_images: image %d, op %d: FLIP_H width %g is not the canvas width %lld", b, i, op.a0, cw);
      ox += sx * (cw - 1); sx = -sx;
      const long long t = vx0; vx0 = cw - vx1; vx1 = cw - t;
    } else if (op.op == SSDK_BOXOP_FLIP_V) {
      SSDK_REQUIRE(op.a0 == (double)ch, "ssdk_assemble_images: image %d, op %d: FLIP_V height %g is not the canvas height %lld", b, i, op.a0, ch);
      oy += sy * (ch - 1); sy = -sy;
      const long long t = vy0; vy0 = ch - vy1; vy1 = ch - t;
    } else {
      SSDK_REQUIRE(op.a0 == (double)ch && op.a1 == (double)cw, "ssdk_assemble_images: image %d, op %d: RESIZE from %gx%g, but the canvas "
                   "is %lldx%lld at that point", b, i, op.a0, op.a1, ch, cw);
      SSDK_REQUIRE(is_int(op.a2) && is_int(op.a3) && op.a2 > 0 && op.a3 > 0, "ssdk_assemble_images: image %d, op %d: RESIZE needs a "
                   "positive integer output size", b, i);
      const int interp = (op.flags >> 8) & 255;
      SSDK_REQUIRE(interp == 0 || interp == 1, "ssdk_assemble_images: image %d, op %d: interpolation mode %d is not supported "
                   "(INTER_NEAREST = 0 and INTER_LINEAR = 1 are)", b, i, interp);
      resized = true; rh = (long long)op.a2; rw = (long long)op.a3;
      mode = interp == 0 ? kImgNearest : kImgLinear;
    }
  }
  const long long fh = resized ? rh : ch, fw = resized ? rw : cw;
  SSDK_REQUIRE(fh == out_h && fw == out_w, "ssdk_assemble_images: image %d ends as %lldx%lld, the output is %dx%d", b, fh, fw, out_h, out_w);
  SSDK_REQUIRE(std::llabs(oy) + ch < (1LL << 30) && std::llabs(ox) + cw < (1LL << 30), "ssdk_assemble_images: image %d: canvas too large", b);
  if (!resized || (rh == ch && rw == cw)) mode = kImgCopy;           // cv2.resize to the same size is a copy
  else if (mode == kImgLinear && ch == 2 * rh && cw == 2 * rw) mode = kImgArea2;
  ImgDesc& d = *out;
  d.src_off = offs[b]; d.h = h; d.w = w; d.c = c;
  d.ch = (int)ch; d.cw = (int)cw; d.oy = (int)oy; d.sy = sy; d.ox = (int)ox; d.sx = sx;
  d.vy0 = (int)vy0; d.vy1 = (int)vy1; d.vx0 = (int)vx0; d.vx1 = (int)vx1;
  d.bg = bg; d.mode = mode;
  d.scale_y = resized ? 1.0 / ((double)rh / (double)ch) : 1.0;
  d.scale_x = resized ? 1.0 / ((double)rw / (double)cw) : 1.0;
  return SSDK_OK;
}

}  // namespace

extern "C" int ssdk_assemble_images(ssdk_ctx* ctx, const uint8_t* src_dev, const long long* src_offsets_host, const int* src_hwc_host, int B,
                                    const ssdk_box_op* ops_host, int max_ops, int out_h, int out_w, float* out_dev, void* stream_) {
  SSDK_REQUIRE(ctx && src_dev && src_offsets_host && src_hwc_host && out_dev, "ssdk_assemble_images: bad argument");
  SSDK_REQUIRE(B > 0 && B <= 65535, "ssdk_assemble_images: batch size %d out of range [1, 65535]", B);
  SSDK_REQUIRE(out_h > 0 && out_w > 0, "ssdk_assemble_images: output size %dx%d must be positive", out_h, out_w);
  SSDK_REQUIRE(max_ops >= 0 && (max_ops == 0 || ops_host), "ssdk_assemble_images: ops_host is NULL");
  std::vector<ImgDesc> descs(B);
  for (int b = 0; b < B; ++b) {
    const int rc = compose_image(b, src_offsets_host, src_hwc_host, ops_host, max_ops, out_h, out_w, &descs[b]);
    if (rc) return rc;
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  const size_t bytes = sizeof(ImgDesc) * (size_t)B;
  int rc = ctx->ws[4].ensure(bytes);
  if (rc) return rc;
  // descriptors: pinned staging (one buffer of the ring) -> workspace, asynchronous; the host waits only if the upload of the
  // call kImgStages calls ago is still queued
  ssdk_ctx::HostStage& st = ctx->img_stage[ctx->img_stage_next];
  if (!st.done) SSDK_CHECK_CUDA(cudaEventCreateWithFlags(&st.done, cudaEventDisableTiming));
  else SSDK_CHECK_CUDA(cudaEventSynchronize(st.done));
  if (st.bytes < bytes) {
    if (st.ptr) cudaFreeHost(st.ptr);
    st.ptr = nullptr; st.bytes = 0;
    const size_t want = std::max(bytes, (size_t)16384);
    SSDK_CHECK_CUDA(cudaHostAlloc(&st.ptr, want, cudaHostAllocDefault));
    st.bytes = want;
  }
  std::memcpy(st.ptr, descs.data(), bytes);
  SSDK_CHECK_CUDA(cudaMemcpyAsync(ctx->ws[4].ptr, st.ptr, bytes, cudaMemcpyHostToDevice, stream));
  SSDK_CHECK_CUDA(cudaEventRecord(st.done, stream));
  ctx->img_stage_next = (ctx->img_stage_next + 1) % ssdk_ctx::kImgStages;
  image_assemble_kernel<<<dim3(out_h, B), kImgThreads, 0, stream>>>(src_dev, reinterpret_cast<const ImgDesc*>(ctx->ws[4].ptr), out_h, out_w, out_dev);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}
