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
// (INTER_NEAREST / INTER_LINEAR) and uint8 cv2.warpAffine (Translate / Scale / Rotate, geometric_ops.py:233-737) in one launch,
// restated in oracle/imageops.py and oracle/warpops.py; the box half of Translate / Scale / Rotate and BoxFilter's overlap test is in oracle/boxops.py.
//   image_assemble_kernel  one CTA per (output row, image): every output pixel is traced back through the resize to at most
//                          four canvas taps, and each tap through the composed crop / pad / flip map to a source pixel or to
//                          the background colour.  No intermediate image exists.
//   photometric_kernel     the photometric prefix of the op lists (ConvertDataType, Brightness, Contrast, Saturation, Hue,
//                          ConvertColor RGB <-> HSV, ChannelSwap; object_detection_2d_photometric_ops.py), one launch in front of
//                          image_assemble_kernel: uint8 in, uint8 h x w x 3 out, restated in oracle/photoops.py.
// The file is compiled with --fmad=false; the float64 resize coordinates also spell their roundings out (__dmul_rn / __dadd_rn).
#include "common.cuh"
#include "rn.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

using namespace ssdk;

namespace {

constexpr int kBoxThreads = 128;

// cos / sin of angle * (CV_PI / 180) for the angles the ops use, as the C library computes them (cv2.getRotationMatrix2D).
__host__ __device__ inline bool cv_cos_sin(double angle, double& c, double& s) {
  if (angle == 0.0) { c = 1.0; s = 0.0; return true; }
  if (angle == 90.0) { c = 0x1.1a62633145c07p-54; s = 1.0; return true; }
  if (angle == 180.0) { c = -1.0; s = 0x1.1a62633145c07p-53; return true; }
  if (angle == 270.0) { c = -0x1.a79394c9e8a0ap-53; s = -1.0; return true; }
  return false;
}

// cv2.getRotationMatrix2D(center, angle, scale): the centre is a Point2f.  The file is compiled with --fmad=false, so every
// product and sum below is rounded on its own, as in OpenCV's scalar code.
__host__ __device__ inline void cv_rotation_matrix(double cx, double cy, double c, double s, double scale, double M[6]) {
  cx = (double)(float)cx; cy = (double)(float)cy;
  const double alpha = c * scale, beta = s * scale;
  M[0] = alpha; M[1] = beta; M[2] = (1 - alpha) * cx - beta * cy;
  M[3] = -beta; M[4] = alpha; M[5] = beta * cx + (1 - alpha) * cy;
}

// Rotate.__call__'s matrix and output size (object_detection_2d_geometric_ops.py:686-700).
__host__ __device__ inline void rotate_geometry(double h, double w, double c, double s, double M[6], long long& h_new, long long& w_new) {
  cv_rotation_matrix(w / 2, h / 2, c, s, 1.0, M);
  const double cos_a = fabs(M[0]), sin_a = fabs(M[1]);
  w_new = (long long)(h * sin_a + w * cos_a);
  h_new = (long long)(h * cos_a + w * sin_a);
  M[5] += (double)(h_new - (long long)h) / 2;
  M[2] += (double)(w_new - (long long)w) / 2;
}

// Both corners through M as np.dot computes them ((m0*x + m1*y) + m2, each step rounded), then np.round(...).astype(int) stored
// back into the float64 labels: a corner that rounds to -0 is stored as +0 (+ 0.0 does that and leaves every other value alone).
__device__ __forceinline__ void corners(const double M[6], double& x0, double& y0, double& x1, double& y1) {
  const double nx0 = rint((M[0] * x0 + M[1] * y0) + M[2]) + 0.0, ny0 = rint((M[3] * x0 + M[4] * y0) + M[5]) + 0.0;
  const double nx1 = rint((M[0] * x1 + M[1] * y1) + M[2]) + 0.0, ny1 = rint((M[3] * x1 + M[4] * y1) + M[5]) + 0.0;
  x0 = nx0; y0 = ny0; x1 = nx1; y1 = ny1;
}

// np.clip(x, lo, hi) on float64 as NumPy computes it: a NaN passes through (fmin / fmax would return the bound), and x is kept
// when it equals a bound, so np.clip(-0.0, 0, h) is -0.0.
__device__ __forceinline__ double np_clip(double x, double lo, double hi) {
  x = x < lo ? lo : x;
  return x > hi ? hi : x;
}

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
            y0 = np_clip(y0, 0.0, op.a2 - 1); y1 = np_clip(y1, 0.0, op.a2 - 1);
            x0 = np_clip(x0, 0.0, op.a3 - 1); x1 = np_clip(x1, 0.0, op.a3 - 1);
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
        } else if (op.op == SSDK_BOXOP_TRANSLATE) {          // labels[:, [xmin, xmax]] += dx_abs; labels[:, [ymin, ymax]] += dy_abs
          x0 += op.a1; x1 += op.a1; y0 += op.a0; y1 += op.a0;
        } else if (op.op == SSDK_BOXOP_SCALE) {
          double M[6];
          cv_rotation_matrix(op.a2 / 2, op.a1 / 2, 1.0, 0.0, op.a0, M);
          corners(M, x0, y0, x1, y1);
        } else if (op.op == SSDK_BOXOP_ROTATE) {
          double M[6], c, s;
          long long hn, wn;
          if (cv_cos_sin(op.a0, c, s) && op.a0 != 0.0) {
            rotate_geometry(op.a1, op.a2, c, s, M, hn, wn);
            corners(M, x0, y0, x1, y1);
            if (op.a0 != 270.0) { const double t = y0; y0 = y1; y1 = t; }   // 90, 180: ymin and ymax were switched
            if (op.a0 != 90.0) { const double t = x0; x0 = x1; x1 = t; }    // 180, 270: xmin and xmax were switched
          }
        } else if (op.op == SSDK_BOXOP_OVERLAP) {            // BoxFilter's overlap test against an a2 x a3 image
          const int crit = op.flags & 3, bp = (op.flags >> 2) & 3;
          const double d = bp == 1 ? 1.0 : bp == 2 ? -1.0 : 0.0, H = op.a2, W = op.a3, lower = op.a0, upper = op.a1;
          if (crit == 0) {
            const double cy = (y0 + y1) / 2, cx = (x0 + x1) / 2;
            valid = valid && (cy >= 0.0) && (cy <= H - 1) && (cx >= 0.0) && (cx <= W - 1);
          } else if (crit == 1) {
            const double area = (x1 - x0 + d) * (y1 - y0 + d);
            const double inter = (np_clip(x1, 0.0, W - 1) - np_clip(x0, 0.0, W - 1) + d) *
                                 (np_clip(y1, 0.0, H - 1) - np_clip(y0, 0.0, H - 1) + d);
            const bool lo = lower == 0.0 ? inter > lower * area : inter >= lower * area;
            valid = valid && lo && (inter <= upper * area);
          } else {                                           // iou(image, box): the intersection ignores border_pixels
            const double iw = fmax(0.0, fmin(W, x1) - fmax(0.0, x0)), ih = fmax(0.0, fmin(H, y1) - fmax(0.0, y0));
            const double inter = iw * ih;
            const double ap = (W - 0.0 + d) * (H - 0.0 + d), aq = (x1 - x0 + d) * (y1 - y0 + d);
            const double v = inter / ((ap + aq) - inter);
            valid = valid && (v > lower) && (v <= upper);
          }
        } else if (op.op == SSDK_BOXOP_CLIP) {               // np.clip to [0, h-1] / [0, w-1]
          y0 = np_clip(y0, 0.0, op.a0 - 1); y1 = np_clip(y1, 0.0, op.a0 - 1);
          x0 = np_clip(x0, 0.0, op.a1 - 1); x1 = np_clip(x1, 0.0, op.a1 - 1);
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
  int rc = ctx->box_ws.ensure(need);
  if (rc) return rc;
  float* tmp = reinterpret_cast<float*>(ctx->box_ws.ptr);
  int* counts = reinterpret_cast<int*>(reinterpret_cast<unsigned char*>(ctx->box_ws.ptr) + (((size_t)(total_in > 0 ? total_in : 1) * 5 * sizeof(float) + 255) / 256 * 256));
  rc = launch(ctx, box_ops_kernel, B, kBoxThreads, 0, stream, gt_in_dev, gt_in_f64, offsets_in_dev, ops_dev, max_ops, tmp, counts);
  if (rc) return rc;
  rc = launch(ctx, box_offsets_kernel, 1, 1024, 0, stream, counts, B, offsets_out_dev, out_stats_dev);
  if (rc) return rc;
  return launch(ctx, box_pack_kernel, B, kBoxThreads, 0, stream, tmp, offsets_in_dev, offsets_out_dev, gt_out_dev);
}

// ------------------------------------------------------------------------------------------------
// Images
// ------------------------------------------------------------------------------------------------
namespace {

constexpr int kImgThreads = 128;
enum { kImgCopy = 0, kImgNearest = 1, kImgLinear = 2, kImgArea2 = 3, kImgWarp = 4 };

// An integer map from a canvas to the image it is drawn from: canvas (r, c) -> (o0 + m00 * r + m01 * c, o1 + m10 * r + m11 * c),
// a translation and a signed axis permutation.  Canvas rows [v0, v1) x columns [v2, v3) come from that image; every other canvas
// pixel shows the background colour.  Crops, pads, flips, translations and 90-degree rotations all compose into one.
struct IntMap {
  int o0, o1, m00, m01, m10, m11;
  int v0, v1, v2, v3;
};

// One image's op list, composed on the host: the integer ops before the resampling step (RESIZE or SCALE) map the canvas it
// reads to the source; the integer ops after a SCALE map the output to the SCALE's output.
struct ImgDesc {
  long long src_off;           // byte offset of the image in the packed source buffer
  int h, w, c;                 // source geometry (c = 1, 3 or 4)
  int ch, cw;                  // canvas size before the resampling step
  IntMap pre;                  // canvas -> source
  IntMap post;                 // output -> SCALE output (kImgWarp only)
  int bg;                      // background R | G << 8 | B << 16
  int mode;                    // kImgCopy / kImgNearest / kImgLinear / kImgArea2 / kImgWarp
  double scale_y, scale_x;     // RESIZE: cv2's 1 / (out / in), float64
  double m[6];                 // SCALE: cv2's inverted matrix, float64
};

__device__ __forceinline__ void bg_px(const ImgDesc& d, int v[3]) {
  v[0] = d.bg & 255; v[1] = (d.bg >> 8) & 255; v[2] = (d.bg >> 16) & 255;
}

__device__ __forceinline__ void canvas_px(const uint8_t* __restrict__ src, const ImgDesc& d, int r, int c, int v[3]) {
  const IntMap& m = d.pre;
  if (r >= m.v0 && r < m.v1 && c >= m.v2 && c < m.v3) {
    const int sr = m.o0 + m.m00 * r + m.m01 * c, sc = m.o1 + m.m10 * r + m.m11 * c;
    const uint8_t* p = src + d.src_off + ((long long)sr * d.w + sc) * d.c;
    if (d.c == 1) { v[0] = v[1] = v[2] = p[0]; }              // gray -> RGB by replication, RGBA -> RGB drops alpha
    else { v[0] = p[0]; v[1] = p[1]; v[2] = p[2]; }
  } else {
    bg_px(d, v);
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

// One pixel (row y, column x) of uint8 cv2.warpAffine, INTER_LINEAR, BORDER_CONSTANT (imgwarp.cpp's WarpAffineInvoker and
// remapBilinear): X0 = rint((m1*y + m2)*1024) + 16, adelta = rint(m0*x*1024), X = (X0 + adelta) >> 5; source column X >> 5
// (saturated to int16), fraction X & 31; likewise for rows with m4, m5, m3.  The bilinear weights (32-fy)(32-fx)*32, ... sum to
// 2^15 exactly; a tap outside the canvas reads the border colour (the one background colour of the list).
__device__ __forceinline__ void warp_px(const uint8_t* __restrict__ src, const ImgDesc& d, int y, int x, int v[3]) {
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(d.m[1], (double)y), d.m[2]), 1024.0)) + 16;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(d.m[4], (double)y), d.m[5]), 1024.0)) + 16;
  const int X = (X0 + __double2int_rn(__dmul_rn(__dmul_rn(d.m[0], (double)x), 1024.0))) >> 5;
  const int Y = (Y0 + __double2int_rn(__dmul_rn(__dmul_rn(d.m[3], (double)x), 1024.0))) >> 5;
  const int sx = min(max(X >> 5, -32768), 32767), sy = min(max(Y >> 5, -32768), 32767), fx = X & 31, fy = Y & 31;
  if (sx >= d.cw || sx + 1 < 0 || sy >= d.ch || sy + 1 < 0) { bg_px(d, v); return; }   // all four taps outside
  int p00[3], p01[3], p10[3], p11[3];
  const bool r0 = sy >= 0, r1 = sy + 1 < d.ch, c0 = sx >= 0, c1 = sx + 1 < d.cw;
  if (r0 && c0) canvas_px(src, d, sy, sx, p00); else bg_px(d, p00);
  if (r0 && c1) canvas_px(src, d, sy, sx + 1, p01); else bg_px(d, p01);
  if (r1 && c0) canvas_px(src, d, sy + 1, sx, p10); else bg_px(d, p10);
  if (r1 && c1) canvas_px(src, d, sy + 1, sx + 1, p11); else bg_px(d, p11);
  const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
#pragma unroll
  for (int k = 0; k < 3; ++k) v[k] = (p00[k] * w00 + p01[k] * w01 + p10[k] * w10 + p11[k] * w11 + (1 << 14)) >> 15;
}

// kWarp: the batch has a SCALE; batches without one run an instantiation that carries no warp code (fewer registers).
template <bool kWarp>
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
    } else if (kWarp && d.mode == kImgWarp) {
      // the integer ops after the SCALE pick the pixel of its output, or the background
      const IntMap& q = d.post;
      if (dy >= q.v0 && dy < q.v1 && dx >= q.v2 && dx < q.v3)
        warp_px(src, d, q.o0 + q.m00 * dy + q.m01 * dx, q.o1 + q.m10 * dy + q.m11 * dx, v);
      else
        bg_px(d, v);
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

// ---- the photometric prefix ----
constexpr int kPhotoThreads = 256;
constexpr int kPhotoMaxStages = 16;
constexpr int kPhotoGroupsPerThread = 4;       // groups of 4 pixels a thread takes, when the grid is sized for the largest image

struct PhotoStage { int op; float a; };        // CHANNEL_SWAP keeps its order in op bits 8-13
struct PhotoDesc {
  long long src_off;                           // the image in the packed source buffer
  long long dst_off;                           // its 3-channel result in the scratch buffer, 16-byte aligned
  int n_px, w, c, n_stages;
  PhotoStage st[kPhotoMaxStages];
};

// The aligned 32-bit word at q, of which only the bytes inside the image [lo, hi) may be read (the packed images start and end
// at arbitrary byte offsets); bytes outside read as 0.
__device__ __forceinline__ uint32_t image_word(const uint8_t* q, const uint8_t* lo, const uint8_t* hi) {
  if (q >= lo && q + 4 <= hi) return *reinterpret_cast<const uint32_t*>(q);
  uint32_t v = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (q + k >= lo && q + k < hi) v |= (uint32_t)q[k] << (8 * k);
  return v;
}

__device__ __forceinline__ float clip255(float x) { return fminf(fmaxf(x, 0.f), 255.f); }   // np.clip(x, 0, 255)
__device__ __forceinline__ float pick3(int k, float x0, float x1, float x2) { return k == 0 ? x0 : k == 1 ? x1 : x2; }

// uint8 cv2.cvtColor(COLOR_RGB2HSV): integer code; sdiv[i] = rint((255 << 12) / i), hdiv[i] = rint((180 << 12) / (6 i)).
__device__ __forceinline__ void rgb2hsv_px(float p[3], const int* __restrict__ sdiv, const int* __restrict__ hdiv) {
  const int r = (int)p[0], g = (int)p[1], b = (int)p[2];
  const int v = max(max(r, g), b), d = v - min(min(r, g), b);
  const int s = (d * sdiv[v] + (1 << 11)) >> 12;
  int h = v == r ? g - b : v == g ? b - r + 2 * d : r - g + 4 * d;
  h = (h * hdiv[d] + (1 << 11)) >> 12;
  if (h < 0) h += 180;
  p[0] = (float)h; p[1] = (float)s; p[2] = (float)v;
}

// uint8 cv2.cvtColor(COLOR_HSV2RGB) as OpenCV 4.13 computes it with AVX2: float32, the two inner 1 - s * x fused, every other
// step rounded; the 32-pixel vector loop truncates the result, the scalar loop that finishes a row (`round`) rounds half to even.
__device__ __forceinline__ void hsv2rgb_px(float p[3], bool round) {
  const float s = mul_rn(p[1], 1.0f / 255.0f), v = mul_rn(p[2], 1.0f / 255.0f);
  const float h = mul_rn(p[0], 6.0f / 180.0f);
  const float ps = truncf(h), f = sub_rn(h, ps);
  int sector = (int)ps;                                           // H <= 255, so h < 9
  if (sector >= 6) sector -= 6;
  const float t1 = mul_rn(v, sub_rn(1.f, s));
  const float t2 = mul_rn(v, __fmaf_rn(-s, f, 1.f));
  const float t3 = mul_rn(v, __fmaf_rn(-s, sub_rn(1.f, f), 1.f));
  float r, g, b;
  switch (sector) {
    case 0: r = v; g = t3; b = t1; break;
    case 1: r = t2; g = v; b = t1; break;
    case 2: r = t1; g = v; b = t3; break;
    case 3: r = t1; g = t2; b = v; break;
    case 4: r = t3; g = t1; b = v; break;
    default: r = v; g = t1; b = t2; break;
  }
  const float x[3] = {mul_rn(r, 255.f), mul_rn(g, 255.f), mul_rn(b, 255.f)};
#pragma unroll
  for (int k = 0; k < 3; ++k) p[k] = (float)min(max(round ? __float2int_rn(x[k]) : __float2int_rz(x[k]), 0), 255);
}

// One CTA column per image with photometric ops (blockIdx.y); a thread takes groups of 4 pixels: 4 * c source bytes from aligned
// words (any source alignment), 12 result bytes as three aligned words.  A pixel is carried as three float32 values, which hold
// the uint8 state exactly; the stage list is uniform across the CTA.
__global__ void __launch_bounds__(kPhotoThreads) photometric_kernel(const uint8_t* __restrict__ src, const PhotoDesc* __restrict__ descs,
                                                                    uint8_t* __restrict__ dst) {
  __shared__ int s_sdiv[256], s_hdiv[256];
  __shared__ PhotoDesc s_d;
  if (threadIdx.x < sizeof(PhotoDesc) / 4)
    reinterpret_cast<int*>(&s_d)[threadIdx.x] = reinterpret_cast<const int*>(descs + blockIdx.y)[threadIdx.x];
  {
    const int i = threadIdx.x;                                    // rint(N / i) = (2N + i) / (2i): neither quotient has a tie
    s_sdiv[i] = i ? (2 * (255 << 12) + i) / (2 * i) : 0;
    s_hdiv[i] = i ? (2 * ((180 << 12) / 6) + i) / (2 * i) : 0;
  }
  __syncthreads();
  const int n_px = s_d.n_px, w = s_d.w, c = s_d.c, n_stages = s_d.n_stages;
  const uint8_t* lo = src + s_d.src_off;
  const uint8_t* hi = lo + (size_t)n_px * c;
  uint8_t* out = dst + s_d.dst_off;
  const int groups = (n_px + 3) >> 2;
  const int tail_from = w & ~31;
  for (int grp = blockIdx.x * kPhotoThreads + threadIdx.x; grp < groups; grp += gridDim.x * kPhotoThreads) {
    // 4 * c bytes from lo + 4 * c * grp, through the aligned words that hold them
    const uint8_t* at = lo + (size_t)grp * 4 * c;
    const int sh = (int)(reinterpret_cast<uintptr_t>(at) & 3);
    const uint8_t* q = at - sh;
    uint32_t in[4] = {0, 0, 0, 0};
    uint32_t prev = image_word(q, lo, hi);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (k < c) {
        const uint32_t next = image_word(q + 4 * (k + 1), lo, hi);
        in[k] = __funnelshift_r(prev, next, 8 * sh);
        prev = next;
      }
    }
    float p[4][3];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        // ConvertTo3Channels: gray is replicated, alpha is dropped
        const uint32_t gray = (in[0] >> (8 * j)) & 255u, rgba = (in[j] >> (8 * k)) & 255u;
        const uint32_t rgb = (in[(3 * j + k) >> 2] >> (8 * ((3 * j + k) & 3))) & 255u;
        p[j][k] = (float)(c == 1 ? gray : c == 4 ? rgba : rgb);
      }
    }
    for (int i = 0; i < n_stages; ++i) {
      const int code = s_d.st[i].op;
      const float a = s_d.st[i].a;
      switch (code & 255) {
        case SSDK_BOXOP_TO_UINT8:                                 // np.round(image, 0).astype(uint8); the values are in [0, 255]
#pragma unroll
          for (int j = 0; j < 4; ++j) { p[j][0] = rint_rn(p[j][0]); p[j][1] = rint_rn(p[j][1]); p[j][2] = rint_rn(p[j][2]); }
          break;
        case SSDK_BOXOP_BRIGHTNESS:                               // np.clip(image + delta, 0, 255)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int k = 0; k < 3; ++k) p[j][k] = clip255(add_rn(p[j][k], a));
          }
          break;
        case SSDK_BOXOP_CONTRAST:                                 // np.clip(127.5 + factor * (image - 127.5), 0, 255)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
#pragma unroll
            for (int k = 0; k < 3; ++k) p[j][k] = clip255(add_rn(127.5f, mul_rn(a, sub_rn(p[j][k], 127.5f))));
          }
          break;
        case SSDK_BOXOP_SATURATION:                               // image[:, :, 1] = np.clip(image[:, :, 1] * factor, 0, 255)
#pragma unroll
          for (int j = 0; j < 4; ++j) p[j][1] = clip255(mul_rn(p[j][1], a));
          break;
        case SSDK_BOXOP_HUE:                                      // image[:, :, 0] = (image[:, :, 0] + delta) % 180.0
#pragma unroll
          for (int j = 0; j < 4; ++j) {                           // NumPy's remainder: fmod, then the sign of the divisor
            float m = fmodf(add_rn(p[j][0], a), 180.f);
            if (m < 0.f) m = add_rn(m, 180.f);
            p[j][0] = m;
          }
          break;
        case SSDK_BOXOP_RGB2HSV:
#pragma unroll
          for (int j = 0; j < 4; ++j) rgb2hsv_px(p[j], s_sdiv, s_hdiv);
          break;
        case SSDK_BOXOP_HSV2RGB: {
          const int x0 = (int)(((long long)grp * 4) % w);
#pragma unroll
          for (int j = 0; j < 4; ++j) hsv2rgb_px(p[j], (x0 + j) % w >= tail_from);
          break;
        }
        case SSDK_BOXOP_CHANNEL_SWAP: {                           // image[:, :, order]
          const int o0 = (code >> 8) & 3, o1 = (code >> 10) & 3, o2 = (code >> 12) & 3;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float x0 = p[j][0], x1 = p[j][1], x2 = p[j][2];
            p[j][0] = pick3(o0, x0, x1, x2); p[j][1] = pick3(o1, x0, x1, x2); p[j][2] = pick3(o2, x0, x1, x2);
          }
          break;
        }
        default: break;                                           // TO_FLOAT32: the values are float32 already
      }
    }
    uint32_t o[3] = {0, 0, 0};
#pragma unroll
    for (int m = 0; m < 12; ++m) o[m >> 2] |= (uint32_t)p[m / 3][m % 3] << (8 * (m & 3));
    uint8_t* to = out + (size_t)grp * 12;
    if (grp * 4 + 4 <= n_px) {
      uint32_t* t32 = reinterpret_cast<uint32_t*>(to);
      t32[0] = o[0]; t32[1] = o[1]; t32[2] = o[2];
    } else {                                                      // the last, partial group
      const int nb = (n_px - grp * 4) * 3;
#pragma unroll
      for (int m = 0; m < 9; ++m)
        if (m < nb) to[m] = (uint8_t)(o[m >> 2] >> (8 * (m & 3)));
    }
  }
}

bool is_photo(int code) { return code >= SSDK_BOXOP_TO_FLOAT32 && code <= SSDK_BOXOP_CHANNEL_SWAP; }

// The photometric prefix of image b's op list -> its stages; every check the entry point documents.
int compose_photo(int b, const ssdk_box_op* ops, int max_ops, PhotoDesc* out) {
  bool geometric = false, is_float = false;
  int n = 0;
  for (int i = 0; i < max_ops; ++i) {
    const ssdk_box_op& op = ops[(size_t)b * max_ops + i];
    if (op.op == SSDK_BOXOP_END) break;
    if (!is_photo(op.op)) {
      geometric = geometric || (op.op >= SSDK_BOXOP_CROP_PAD && op.op <= SSDK_BOXOP_ROTATE && op.op != SSDK_BOXOP_FILTER);
      continue;
    }
    SSDK_REQUIRE(!geometric, "ssdk_assemble_images: image %d, op %d: photometric ops must come before every op that changes the "
                 "image geometry", b, i);
    SSDK_REQUIRE(n < kPhotoMaxStages, "ssdk_assemble_images: image %d: more than %d photometric ops", b, kPhotoMaxStages);
    PhotoStage st{op.op, (float)op.a0};
    switch (op.op) {
      case SSDK_BOXOP_TO_FLOAT32: is_float = true; break;
      case SSDK_BOXOP_TO_UINT8: is_float = false; break;
      case SSDK_BOXOP_RGB2HSV: case SSDK_BOXOP_HSV2RGB:
        SSDK_REQUIRE(!is_float, "ssdk_assemble_images: image %d, op %d: a colour conversion needs a uint8 image (TO_UINT8 first)", b, i);
        break;
      case SSDK_BOXOP_CHANNEL_SWAP: {
        const double o[3] = {op.a0, op.a1, op.a2};
        int seen = 0;
        for (double v : o) seen |= (v == 0.0 || v == 1.0 || v == 2.0) ? 1 << (int)v : 8;
        SSDK_REQUIRE(seen == 7, "ssdk_assemble_images: image %d, op %d: CHANNEL_SWAP order (%g, %g, %g) is not a permutation of "
                     "(0, 1, 2)", b, i, op.a0, op.a1, op.a2);
        st.op |= ((int)o[0] << 8) | ((int)o[1] << 10) | ((int)o[2] << 12);
        break;
      }
      default:
        SSDK_REQUIRE(is_float, "ssdk_assemble_images: image %d, op %d: BRIGHTNESS / CONTRAST / SATURATION / HUE need a float32 image "
                     "(TO_FLOAT32 first)", b, i);
        if (op.op == SSDK_BOXOP_BRIGHTNESS)
          SSDK_REQUIRE(std::isfinite(op.a0), "ssdk_assemble_images: image %d, op %d: BRIGHTNESS delta %g is not finite", b, i, op.a0);
        else if (op.op == SSDK_BOXOP_HUE)
          SSDK_REQUIRE(op.a0 >= -180.0 && op.a0 <= 180.0, "`delta` must be in the closed interval `[-180, 180]`. (image %d, op %d: %g)", b, i, op.a0);
        else
          SSDK_REQUIRE(op.a0 > 0.0 && std::isfinite(op.a0), "It must be `factor > 0`. (image %d, op %d: %g)", b, i, op.a0);
    }
    out->st[n++] = st;
  }
  SSDK_REQUIRE(!is_float, "ssdk_assemble_images: image %d: the photometric ops leave a float32 image (TO_UINT8 is missing)", b);
  out->n_stages = n;
  return SSDK_OK;
}

bool is_int(double a) { return a == std::floor(a) && std::fabs(a) <= (double)(1 << 24); }

// Host form of IntMap while a list is composed: canvas h x w, canvas (r, c) -> o + m * (r, c), rows [v0, v1) x cols [v2, v3) valid.
struct HostMap {
  long long h, w, o0, o1, m00, m01, m10, m11, v0, v1, v2, v3;
};
// One integer op: the new canvas is nh x nw, and new (r, c) shows old (t0 + p00 * r + p01 * c, t1 + p10 * r + p11 * c), where
// that lies in the old canvas, the op's background colour elsewhere.  p is a signed permutation.
struct IntOp {
  long long nh, nw, t0, t1;
  int p00, p01, p10, p11;
};

HostMap identity_map(long long h, long long w) { return HostMap{h, w, 0, 0, 1, 0, 0, 1, 0, h, 0, w}; }

// {u : lo <= t + s * u < hi} for s = +-1, as [a, b)
void pre_interval(long long lo, long long hi, long long t, int s, long long& a, long long& b) {
  if (s > 0) { a = lo - t; b = hi - t; } else { a = t - hi + 1; b = t - lo + 1; }
}

// The new-canvas rectangle whose pixels the op draws from the old rectangle rows [r0, r1) x cols [c0, c1).
void preimage(const IntOp& op, long long r0, long long r1, long long c0, long long c1, long long v[4]) {
  if (op.p00 != 0) { pre_interval(r0, r1, op.t0, op.p00, v[0], v[1]); pre_interval(c0, c1, op.t1, op.p11, v[2], v[3]); }
  else { pre_interval(r0, r1, op.t0, op.p01, v[2], v[3]); pre_interval(c0, c1, op.t1, op.p10, v[0], v[1]); }
  v[0] = std::max(v[0], 0LL); v[1] = std::min(v[1], op.nh); v[2] = std::max(v[2], 0LL); v[3] = std::min(v[3], op.nw);
  if (v[1] <= v[0] || v[3] <= v[2]) v[0] = v[1] = v[2] = v[3] = 0;
}

// Compose op into map; returns whether the op brings background into its canvas.
bool compose(HostMap& m, const IntOp& op) {
  long long full[4], v[4];
  preimage(op, 0, m.h, 0, m.w, full);
  preimage(op, m.v0, m.v1, m.v2, m.v3, v);
  HostMap n;
  n.h = op.nh; n.w = op.nw;
  n.o0 = m.o0 + m.m00 * op.t0 + m.m01 * op.t1; n.o1 = m.o1 + m.m10 * op.t0 + m.m11 * op.t1;
  n.m00 = m.m00 * op.p00 + m.m01 * op.p10; n.m01 = m.m00 * op.p01 + m.m01 * op.p11;
  n.m10 = m.m10 * op.p00 + m.m11 * op.p10; n.m11 = m.m10 * op.p01 + m.m11 * op.p11;
  n.v0 = v[0]; n.v1 = v[1]; n.v2 = v[2]; n.v3 = v[3];
  m = n;
  return !(full[0] == 0 && full[1] == op.nh && full[2] == 0 && full[3] == op.nw);
}

IntMap device_map(const HostMap& m) {
  return IntMap{(int)m.o0, (int)m.o1, (int)m.m00, (int)m.m01, (int)m.m10, (int)m.m11, (int)m.v0, (int)m.v1, (int)m.v2, (int)m.v3};
}

// warpAffine's inversion of a forward matrix (imgwarp.cpp; the same as cv2.invertAffineTransform).
void cv_invert_affine(double M[6]) {
  double D = M[0] * M[4] - M[1] * M[3];
  D = D != 0 ? 1. / D : 0;
  const double A11 = M[4] * D, A22 = M[0] * D;
  M[0] = A11; M[1] *= -D;
  M[3] *= -D; M[4] = A22;
  const double b1 = -M[0] * M[2] - M[1] * M[5];
  const double b2 = -M[3] * M[2] - M[4] * M[5];
  M[2] = b1; M[5] = b2;
}

constexpr long long kShortMax = 32767;

// cv2's fixed-point coordinates of a warp to nh x nw with inverse matrix m stay in int32 (the largest magnitude of
// X0 + adelta, linear in the row and the column, is reached at a corner).
bool fixed_point_fits(const double m[6], long long nh, long long nw) {
  for (int k = 0; k < 2; ++k) {
    const double* r = m + 3 * k;
    double worst = 0;
    for (long long y : {0LL, nh - 1})
      for (long long x : {0LL, nw - 1})
        worst = std::max(worst, std::fabs((r[1] * (double)y + r[2]) * 1024.0) + std::fabs(r[0] * (double)x * 1024.0));
    if (!(worst < (double)(1 << 30))) return false;
  }
  return true;
}

// Rotate's warp as an integer op: cv2's fixed-point map (X0(y) + adelta(x), Y0(y) + bdelta(x)) is computed for every output row
// and column and must be exactly 1024 * (a signed permutation of (y, x) plus an integer offset) + 16, so every sample has
// fraction 0 and the warp is a pixel permutation with the border colour (black) where it leaves the source.
bool rotate_op(long long h, long long w, double angle, IntOp& op) {
  double c, s, M[6];
  if (!cv_cos_sin(angle, c, s) || angle == 0.0) return false;
  long long hn, wn;
  rotate_geometry((double)h, (double)w, c, s, M, hn, wn);
  cv_invert_affine(M);
  op.nh = hn; op.nw = wn;
  op.p11 = (int)std::rint(M[0]); op.p10 = (int)std::rint(M[1]); op.t1 = (long long)std::rint(M[2]);
  op.p01 = (int)std::rint(M[3]); op.p00 = (int)std::rint(M[4]); op.t0 = (long long)std::rint(M[5]);
  const bool perm = (op.p00 != 0 && op.p01 == 0 && op.p10 == 0 && op.p11 != 0) || (op.p00 == 0 && op.p01 != 0 && op.p10 != 0 && op.p11 == 0);
  if (!perm || hn <= 0 || wn <= 0 || !fixed_point_fits(M, hn, wn)) return false;
  for (long long x = 0; x < wn; ++x) {
    if (std::nearbyint(M[0] * (double)x * 1024.0) != (double)(1024 * op.p11 * x)) return false;
    if (std::nearbyint(M[3] * (double)x * 1024.0) != (double)(1024 * op.p01 * x)) return false;
  }
  for (long long y = 0; y < hn; ++y) {
    if (std::nearbyint((M[1] * (double)y + M[2]) * 1024.0) != (double)(1024 * (op.t1 + op.p10 * y))) return false;
    if (std::nearbyint((M[4] * (double)y + M[5]) * 1024.0) != (double)(1024 * (op.t0 + op.p00 * y))) return false;
  }
  return true;
}

// Compose image b's op list into its descriptor; every check the entry point documents.
int compose_image(int b, const long long* offs, const int* hwc, const ssdk_box_op* ops, int max_ops, int out_h, int out_w, ImgDesc* out) {
  const int h = hwc[3 * b], w = hwc[3 * b + 1], c = hwc[3 * b + 2];
  SSDK_REQUIRE(h > 0 && w > 0, "ssdk_assemble_images: image %d has size %dx%d", b, h, w);
  SSDK_REQUIRE(c == 1 || c == 3 || c == 4, "ssdk_assemble_images: image %d has %d channels (1, 3 or 4 are supported)", b, c);
  SSDK_REQUIRE(offs[b] >= 0 && offs[b + 1] - offs[b] == (long long)h * w * c,
               "ssdk_assemble_images: image %d: offsets %lld..%lld do not hold %dx%dx%d bytes", b, offs[b], offs[b + 1], h, w, c);
  HostMap pre = identity_map(h, w), post = identity_map(0, 0);
  HostMap* cur = &pre;                                            // the map the next integer op composes into
  int bg = 0, mode = kImgCopy;
  bool has_bg = false, resized = false, warped = false;
  long long rh = 0, rw = 0;
  double minv[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < max_ops; ++i) {
    const ssdk_box_op& op = ops[(size_t)b * max_ops + i];
    if (op.op == SSDK_BOXOP_END) break;
    if (op.op == SSDK_BOXOP_FILTER || op.op == SSDK_BOXOP_OVERLAP || op.op == SSDK_BOXOP_CLIP) continue;   // boxes only
    if (is_photo(op.op)) continue;                                  // run by photometric_kernel (compose_photo)
    SSDK_REQUIRE(op.op >= SSDK_BOXOP_CROP_PAD && op.op <= SSDK_BOXOP_ROTATE, "ssdk_assemble_images: image %d, op %d: unknown op code %d", b, i, op.op);
    SSDK_REQUIRE(!resized, "ssdk_assemble_images: image %d, op %d: the RESIZE must be the last op that changes the image", b, i);
    const long long ch = cur->h, cw = cur->w;
    const int col = (int)(((unsigned)op.flags >> 8) & 0xFFFFFFu);
    IntOp io{ch, cw, 0, 0, 1, 0, 0, 1};
    int io_bg = col;
    if (op.op == SSDK_BOXOP_CROP_PAD) {
      SSDK_REQUIRE(is_int(op.a0) && is_int(op.a1) && is_int(op.a2) && is_int(op.a3) && op.a2 > 0 && op.a3 > 0,
                   "ssdk_assemble_images: image %d, op %d: CROP_PAD needs an integer patch of positive size", b, i);
      const long long py = (long long)op.a0, px = (long long)op.a1;
      SSDK_REQUIRE(!(py > ch || px > cw), "The given patch doesn't overlap with the input image. (image %d, op %d)", b, i);
      io.nh = (long long)op.a2; io.nw = (long long)op.a3; io.t0 = py; io.t1 = px;
    } else if (op.op == SSDK_BOXOP_FLIP_H) {
      SSDK_REQUIRE(op.a0 == (double)cw, "ssdk_assemble_images: image %d, op %d: FLIP_H width %g is not the canvas width %lld", b, i, op.a0, cw);
      io.t1 = cw - 1; io.p11 = -1;
    } else if (op.op == SSDK_BOXOP_FLIP_V) {
      SSDK_REQUIRE(op.a0 == (double)ch, "ssdk_assemble_images: image %d, op %d: FLIP_V height %g is not the canvas height %lld", b, i, op.a0, ch);
      io.t0 = ch - 1; io.p00 = -1;
    } else if (op.op == SSDK_BOXOP_TRANSLATE) {
      SSDK_REQUIRE(op.a2 == (double)ch && op.a3 == (double)cw, "ssdk_assemble_images: image %d, op %d: TRANSLATE of a %gx%g image, but the "
                   "canvas is %lldx%lld at that point", b, i, op.a2, op.a3, ch, cw);
      SSDK_REQUIRE(is_int(op.a0) && is_int(op.a1) && std::fabs(op.a0) < (double)(1 << 20) && std::fabs(op.a1) < (double)(1 << 20),
                   "ssdk_assemble_images: image %d, op %d: TRANSLATE needs integer shifts below 2^20 pixels", b, i);
      io.t0 = -(long long)op.a0; io.t1 = -(long long)op.a1;       // warpAffine with an integer matrix: a shift, fraction 0
    } else if (op.op == SSDK_BOXOP_ROTATE) {
      SSDK_REQUIRE(op.a0 == 90.0 || op.a0 == 180.0 || op.a0 == 270.0, "ssdk_assemble_images: image %d, op %d: ROTATE angle %g is not "
                   "90, 180 or 270", b, i, op.a0);
      SSDK_REQUIRE(op.a1 == (double)ch && op.a2 == (double)cw, "ssdk_assemble_images: image %d, op %d: ROTATE of a %gx%g image, but the "
                   "canvas is %lldx%lld at that point", b, i, op.a1, op.a2, ch, cw);
      SSDK_REQUIRE(ch < kShortMax && cw < kShortMax, "ssdk_assemble_images: image %d, op %d: ROTATE of a %lldx%lld canvas (cv2's warp "
                   "needs sides below 32767)", b, i, ch, cw);
      SSDK_REQUIRE(rotate_op(ch, cw, op.a0, io), "ssdk_assemble_images: image %d, op %d: cv2's fixed-point map of this ROTATE is not an "
                   "exact pixel permutation", b, i);
      io_bg = 0;                                                  // Rotate's warpAffine keeps cv2's default border: black
    } else {
      const bool scale = op.op == SSDK_BOXOP_SCALE;
      SSDK_REQUIRE(!warped, "ssdk_assemble_images: image %d, op %d: at most one resampling step (RESIZE or SCALE) per list", b, i);
      if (!scale) {
        SSDK_REQUIRE(op.a0 == (double)ch && op.a1 == (double)cw, "ssdk_assemble_images: image %d, op %d: RESIZE from %gx%g, but the canvas "
                     "is %lldx%lld at that point", b, i, op.a0, op.a1, ch, cw);
        SSDK_REQUIRE(is_int(op.a2) && is_int(op.a3) && op.a2 > 0 && op.a3 > 0, "ssdk_assemble_images: image %d, op %d: RESIZE needs a "
                     "positive integer output size", b, i);
        const int interp = (op.flags >> 8) & 255;
        SSDK_REQUIRE(interp == 0 || interp == 1, "ssdk_assemble_images: image %d, op %d: interpolation mode %d is not supported "
                     "(INTER_NEAREST = 0 and INTER_LINEAR = 1 are)", b, i, interp);
        resized = true; rh = (long long)op.a2; rw = (long long)op.a3;
        mode = interp == 0 ? kImgNearest : kImgLinear;
        continue;
      }
      SSDK_REQUIRE(op.a1 == (double)ch && op.a2 == (double)cw, "ssdk_assemble_images: image %d, op %d: SCALE of a %gx%g image, but the "
                   "canvas is %lldx%lld at that point", b, i, op.a1, op.a2, ch, cw);
      SSDK_REQUIRE(op.a0 > 0 && std::isfinite(op.a0), "ssdk_assemble_images: image %d, op %d: SCALE factor %g is not positive", b, i, op.a0);
      SSDK_REQUIRE(ch < kShortMax && cw < kShortMax, "ssdk_assemble_images: image %d, op %d: SCALE of a %lldx%lld canvas (cv2's warp "
                   "needs sides below 32767)", b, i, ch, cw);
      cv_rotation_matrix((double)cw / 2, (double)ch / 2, 1.0, 0.0, op.a0, minv);
      cv_invert_affine(minv);
      SSDK_REQUIRE(fixed_point_fits(minv, ch, cw), "ssdk_assemble_images: image %d, op %d: SCALE factor %g overflows cv2's fixed-point "
                   "coordinates", b, i, op.a0);
      SSDK_REQUIRE(!has_bg || col == bg, "ssdk_assemble_images: image %d, op %d: ops with different background colours in one list are "
                   "not supported", b, i);
      has_bg = true; bg = col;
      warped = true; mode = kImgWarp;
      post = identity_map(ch, cw);
      cur = &post;
      continue;
    }
    if (compose(*cur, io)) {                                      // the op brings in background
      SSDK_REQUIRE(!has_bg || io_bg == bg, "ssdk_assemble_images: image %d, op %d: ops with different background colours in one list "
                   "are not supported", b, i);
      has_bg = true; bg = io_bg;
    }
  }
  const long long ch = pre.h, cw = pre.w;
  const long long fh = resized ? rh : warped ? post.h : ch, fw = resized ? rw : warped ? post.w : cw;
  SSDK_REQUIRE(fh == out_h && fw == out_w, "ssdk_assemble_images: image %d ends as %lldx%lld, the output is %dx%d", b, fh, fw, out_h, out_w);
  for (const HostMap* m : {&pre, &post})
    SSDK_REQUIRE(std::llabs(m->o0) + m->h + m->w < (1LL << 30) && std::llabs(m->o1) + m->h + m->w < (1LL << 30),
                 "ssdk_assemble_images: image %d: canvas too large", b);
  if (resized && rh == ch && rw == cw) mode = kImgCopy;            // cv2.resize to the same size is a copy
  else if (mode == kImgLinear && ch == 2 * rh && cw == 2 * rw) mode = kImgArea2;
  ImgDesc& d = *out;
  d.src_off = offs[b]; d.h = h; d.w = w; d.c = c;
  d.ch = (int)ch; d.cw = (int)cw;
  d.pre = device_map(pre); d.post = device_map(post);
  d.bg = bg; d.mode = mode;
  d.scale_y = resized ? 1.0 / ((double)rh / (double)ch) : 1.0;
  d.scale_x = resized ? 1.0 / ((double)rw / (double)cw) : 1.0;
  for (int k = 0; k < 6; ++k) d.m[k] = minv[k];
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
  std::vector<PhotoDesc> photo;                                   // the images with photometric ops
  std::vector<int> photo_image;
  long long photo_bytes = 0;
  int photo_groups = 0;
  for (int b = 0; b < B; ++b) {
    PhotoDesc p{};
    int rc = compose_photo(b, ops_host, max_ops, &p);
    if (rc) return rc;
    rc = compose_image(b, src_offsets_host, src_hwc_host, ops_host, max_ops, out_h, out_w, &descs[b]);
    if (rc) return rc;
    if (!p.n_stages) continue;
    const long long n_px = (long long)descs[b].h * descs[b].w;
    SSDK_REQUIRE(n_px < (1LL << 31) - 4, "ssdk_assemble_images: image %d is too large for the photometric ops", b);
    p.src_off = descs[b].src_off; p.dst_off = photo_bytes;
    p.n_px = (int)n_px; p.w = descs[b].w; p.c = descs[b].c;
    photo_bytes += (n_px * 3 + 15) / 16 * 16;
    photo_groups = std::max(photo_groups, (int)((n_px + 3) / 4));
    photo.push_back(p); photo_image.push_back(b);
  }
  cudaStream_t stream = (cudaStream_t)stream_;
  const size_t img_bytes = sizeof(ImgDesc) * (size_t)B;
  const size_t bytes = img_bytes + sizeof(PhotoDesc) * photo.size();
  int rc = ctx->img_desc_ws.ensure(bytes);
  if (rc) return rc;
  if (!photo.empty()) {
    rc = ctx->photo_ws.ensure((size_t)photo_bytes);
    if (rc) return rc;
    // image_assemble_kernel addresses every image as src_dev + src_off: the images in the scratch buffer get their distance
    // from src_dev (both are device addresses of one flat address space)
    for (size_t k = 0; k < photo.size(); ++k) {
      ImgDesc& d = descs[photo_image[k]];
      d.src_off = (long long)(reinterpret_cast<uintptr_t>(ctx->photo_ws.ptr) + (uintptr_t)photo[k].dst_off) - (long long)reinterpret_cast<uintptr_t>(src_dev);
      d.c = 3;
    }
  }
  // descriptors: pinned staging -> workspace, asynchronous; the host waits only if the upload from the same staging buffer,
  // four calls ago, is still queued
  rc = ctx->img_desc_ring.upload(ctx->img_desc_ws.ptr, stream, {{descs.data(), img_bytes}, {photo.data(), bytes - img_bytes}});
  if (rc) return rc;
  const ImgDesc* d_dev = reinterpret_cast<const ImgDesc*>(ctx->img_desc_ws.ptr);
  if (!photo.empty()) {
    const int gx = std::max(1, std::min(ceil_div(photo_groups, kPhotoThreads * kPhotoGroupsPerThread), 65535));
    rc = launch(ctx, photometric_kernel, dim3(gx, (unsigned)photo.size()), kPhotoThreads, 0, stream,
                src_dev, reinterpret_cast<const PhotoDesc*>(static_cast<const unsigned char*>(ctx->img_desc_ws.ptr) + img_bytes),
                static_cast<uint8_t*>(ctx->photo_ws.ptr));
    if (rc) return rc;
  }
  const bool warp = std::any_of(descs.begin(), descs.end(), [](const ImgDesc& d) { return d.mode == kImgWarp; });
  return launch(ctx, warp ? image_assemble_kernel<true> : image_assemble_kernel<false>, dim3(out_h, B), kImgThreads, 0, stream,
                src_dev, d_dev, out_h, out_w, out_dev);
}
