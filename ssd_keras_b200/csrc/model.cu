// Static execution plan for the SSD graphs (models/keras_ssd300.py:263-419, keras_ssd512.py, keras_ssd7.py:266-393).
// The host (Python, mirroring the reference builders) describes the graph layer by layer; this file sizes the
// zero-bordered activation buffers, packs the weights into K-major bf16 hi/lo planes on the device, builds the TMA descriptors
// and tile lists once, and replays the kernel sequence on every forward call.
#include "model.cuh"
#include <memory>

using namespace ssdk;

namespace {

// fp32 master kernel, HWIO [taps][cin][cout], and bias of a conv layer.  A head fuses its conf and loc kernels (and biases) per
// box as [C logits | 4 offsets], the order of its output channels; every packed weight plane is made from this master.
void fused_master(const ssdk_layer_desc& d, int cin, int cout, int Ctot, std::vector<float>& w, std::vector<float>& bias) {
  const size_t K = (size_t)d.kh * d.kw * cin;
  w.assign(K * cout, 0.f);
  bias.assign(cout, 0.f);
  for (int o = 0; o < cout; ++o) {
    const float* ker = d.kernel; const float* b = d.bias;
    int oc = o, ocn = cout;                             // column of `ker`, and its number of columns
    if (d.op == SSDK_OP_HEAD) {
      const int box = o / (Ctot + 4), r = o % (Ctot + 4);
      if (r < Ctot) { oc = box * Ctot + r; ocn = d.n_boxes * Ctot; }
      else { ker = d.kernel2; b = d.bias2; oc = box * 4 + (r - Ctot); ocn = d.n_boxes * 4; }
    }
    if (b) bias[o] = b[oc];
    for (size_t k = 0; k < K; ++k) w[k * cout + o] = ker[k * ocn + oc];
  }
}

struct CudaFree { void operator()(void* p) const { cudaFree(p); } };

int build_conv(ssdk_model* m, int li) {
  LayerPlan& L = m->layers[li];
  const ssdk_layer_desc& d = L.d;
  const LayerPlan& in = m->layers[d.input];
  const ActBuf& ia = in.out;
  const int cin = in.C;
  const bool head = d.op == SSDK_OP_HEAD;
  const int cout = head ? d.n_boxes * (m->Ctot + 4) : d.cout;
  const int taps = d.kh * d.kw;
  SSDK_REQUIRE(taps <= kMaxTaps, "conv kernel %dx%d is larger than the supported %d taps", d.kh, d.kw, kMaxTaps);
  SSDK_REQUIRE(head || cout % 8 == 0, "conv output channels must be a multiple of 8 (got %d)", cout);
  L.direct = !head && cin <= 4 && d.stride == 1 && cout % 16 == 0 && (size_t)taps * cin * cout * 4 <= 96 * 1024 && ia.Cs == 8;
  std::vector<float> master, bias;
  fused_master(d, cin, cout, m->Ctot, master, bias);
  // conv + BatchNormalization in a training plan: the conv writes its raw output z, batch statistics follow (bn.cu)
  L.bn_train = m->training && !head && d.bn_gamma && d.bn_beta && d.bn_mean && d.bn_var;
  if (L.bn_train) {
    int rc = alloc_act(m, L.z, m->B, L.H, L.W, L.C, 0); if (rc) return rc;
    rc = upload_f32(m, &L.bn_gamma, d.bn_gamma, cout); if (rc) return rc;
    rc = upload_f32(m, &L.bn_beta, d.bn_beta, cout); if (rc) return rc;
    rc = upload_f32(m, &L.bn_mmean, d.bn_mean, cout); if (rc) return rc;
    rc = upload_f32(m, &L.bn_mvar, d.bn_var, cout); if (rc) return rc;
    rc = dev_alloc(m->allocs, &L.bn_bmean, cout, true); if (rc) return rc;
    rc = dev_alloc(m->allocs, &L.bn_brstd, cout, true); if (rc) return rc;
    rc = dev_alloc(m->allocs, &L.bn_acc, (size_t)2 * cout, true); if (rc) return rc;
    L.bn_eps = d.bn_eps > 0.f ? d.bn_eps : 1e-3f;
    L.bn_momentum = (d.bn_momentum > 0.f && d.bn_momentum < 1.f) ? d.bn_momentum : 0.99f;
  }
  // experiment knob (inference plans only): route the image-facing layer through im2col (K = 27 -> 32) + the implicit GEMM instead
  if (L.direct && !m->training && getenv("SSDK_NO_DIRECT")) L.direct = false;
  if (L.direct) {
    int rc = upload_f32(m, &L.w_f32, master.data(), master.size()); if (rc) return rc;
    rc = upload_f32(m, &L.bias, bias.data(), bias.size()); if (rc) return rc;
    if (d.bn_scale && d.bn_shift && !L.bn_train) {
      rc = upload_f32(m, &L.bn_scale, d.bn_scale, cout); if (rc) return rc;
      rc = upload_f32(m, &L.bn_shift, d.bn_shift, cout); if (rc) return rc;
    }
    const double fl = 2.0 * m->B * L.H * L.W * (double)taps * cin * cout;
    m->flops_algo += fl;                 // counted as algorithmic FLOPs only (the timed conv launches exclude this layer)
    // inference plans: the layer runs on the tensor cores with a gathered A tile (conv_first_kernel); training plans keep the fp32
    // direct kernel, whose weights are the optimizer's master copy
    if (!m->training && first_tc_supported(taps, cin, cout) && d.dilation >= 1 && first_border_ok(ia, d.kh, d.kw, d.dilation, d.pad_t, d.pad_l) &&
        !getenv("SSDK_NO_FIRST_TC")) {
      std::vector<uint16_t> whi, wlo;
      L.first = first_plan(L.out, d.kh, d.kw, m->ctx->sm_count);
      first_weight_image(master.data(), taps, cin, cout, L.first.BN, L.first.kblocks, whi, wlo);
      rc = dev_alloc(m->allocs, &L.w_hi, whi.size(), false); if (rc) return rc;
      SSDK_CHECK_CUDA(cudaMemcpy(L.w_hi, whi.data(), whi.size() * 2, cudaMemcpyHostToDevice));
      if (m->split) {
        rc = dev_alloc(m->allocs, &L.w_lo, wlo.size(), false); if (rc) return rc;
        SSDK_CHECK_CUDA(cudaMemcpy(L.w_lo, wlo.data(), wlo.size() * 2, cudaMemcpyHostToDevice));
      }
      L.first_tc = true;
    }
    return SSDK_OK;
  }
  L.im2col = (d.stride != 1) || (cin < 8);
  ConvLaunch& cl = L.launch;
  ConvArgs& a = cl.args;
  const int Ho = L.H, Wo = L.W;
  ConvGeom g;
  g.Ho = Ho; g.Wo = Wo; g.B = m->B; g.cout = cout;
  int kblocks;
  if (L.im2col) {
    L.Kpad = (taps * cin + 7) / 8 * 8;
    kblocks = (L.Kpad + 63) / 64;
    size_t n = (size_t)m->B * Ho * Wo * L.Kpad + 64 * 8;
    int rc = dev_alloc(m->allocs, &L.col_hi, n, true); if (rc) return rc;
    if (m->split) { rc = dev_alloc(m->allocs, &L.col_lo, n, true); if (rc) return rc; }
    L.im2col_vec8 = im2col_vec8_ok(ia, L.Kpad, L.col_hi, L.col_lo);
    g.a_hi = L.col_hi; g.a_lo = L.col_lo; g.a_inner = L.Kpad; g.a_rows = (uint64_t)m->B * Ho * Wo;
  } else {
    kblocks = (ia.Cs + 63) / 64;
    g.in = &ia; g.kh = d.kh; g.kw = d.kw; g.dilation = d.dilation; g.pad_t = d.pad_t; g.pad_l = d.pad_l;
    SSDK_REQUIRE(ia.pad >= std::max(std::max(d.pad_t, d.pad_b), std::max(d.pad_l, d.pad_r)), "internal: activation border too small");
  }
  L.kblocks = kblocks;
  // weights: forward planes packed on the device from the master, which training plans keep for the optimiser
  L.w_krow = L.im2col ? (size_t)kblocks * 64 : (size_t)taps * kblocks * 64;
  int rc = dev_alloc(m->allocs, &L.w_hi, (size_t)cout * L.w_krow, false); if (rc) return rc;
  if (m->split) { rc = dev_alloc(m->allocs, &L.w_lo, (size_t)cout * L.w_krow, false); if (rc) return rc; }
  std::unique_ptr<float, CudaFree> scratch;         // the master of an inference plan, freed once the planes are packed
  float* w_dev = nullptr;
  if (m->training) {
    rc = upload_f32(m, &L.w_f32, master.data(), master.size()); if (rc) return rc;
    w_dev = L.w_f32;
  } else {
    SSDK_CHECK_CUDA(cudaMalloc(&w_dev, master.size() * sizeof(float)));
    scratch.reset(w_dev);
    SSDK_CHECK_CUDA(cudaMemcpy(w_dev, master.data(), master.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  rc = launch_repack(m->ctx, w_dev, taps, cin, cout, L.im2col ? PACK_FWD_IM2COL : PACK_FWD, kblocks, L.w_krow, L.w_hi, L.w_lo, 0);
  if (rc) return rc;
  rc = plan_conv_gemm(m, cl, g, L.w_hi, L.w_lo, L.w_krow, kblocks, &L.tile_list);
  if (rc) return rc;
  rc = upload_f32(m, &L.bias, bias.data(), bias.size()); if (rc) return rc;
  a.bias = L.bias;
  if (d.bn_scale && d.bn_shift && !head && !L.bn_train) {
    rc = upload_f32(m, &L.bn_scale, d.bn_scale, cout); if (rc) return rc;
    rc = upload_f32(m, &L.bn_shift, d.bn_shift, cout); if (rc) return rc;
    a.bn_scale = L.bn_scale; a.bn_shift = L.bn_shift;
  }
  a.act = L.bn_train ? SSDK_ACT_NONE : d.act;
  if (head) {
    // inference plans: softmax / concat / anchors in the epilogue, straight into y_pred (one n-tile holds all boxes of a pixel);
    // training plans keep the raw logits (the backward pass needs them) and finish with head_finalize_kernel
    const bool fuse = !m->training && a.n_tiles_n == 1 && !getenv("SSDK_NO_HEAD_FUSION");
    if (fuse) {
      a.epi = EPI_HEAD;
      a.head_nb = d.n_boxes; a.head_C = m->Ctot; a.head_prior_off = 0;          // prior offset, P, anchors: set once they are known
      L.head_fused = true;
    } else {
      a.epi = EPI_F32;
      rc = dev_alloc(m->allocs, &L.head_f32, (size_t)m->B * Ho * Wo * cout, true); if (rc) return rc;
      a.out_f32 = L.head_f32;
    }
  } else {
    a.epi = EPI_SPLIT;
    const ActBuf& dst = L.bn_train ? L.z : L.out;
    a.out_hi = dst.hi; a.out_lo = dst.lo; a.out_Hp = dst.Hp(); a.out_Wp = dst.Wp(); a.out_pad = dst.pad; a.out_Cs = dst.Cs;
  }
  cl.flops_algo = 2.0 * m->B * Ho * Wo * (double)taps * cin * cout;
  m->flops_algo += cl.flops_algo; m->flops_issued += cl.flops_issued;
  return SSDK_OK;
}


// Two-stream schedule for inference plans.  The tail of an SSD trunk (conv7_1 ... conv9_2 at batch 32) and the predictor heads on
// the small feature maps are launches of 3 ... 36 CTAs that each wait out their own TMA / MMA latency chain while >100 SMs idle;
// the predictor heads on the large maps are wide but independent of that tail.  From the first trunk convolution after which every
// trunk convolution is narrow (grid <= R), narrow launches go to a second stream and the wide ones stay on the caller's stream with
// their persistent grid capped at sm_count - (widest narrow grid), so both sets always find free SMs (every conv CTA owns an SM:
// ~200 KB of shared memory).  Cross-stream dependencies are events recorded at issue time; the streams join before the call returns.
// SSDK_OVERLAP=0 disables, SSDK_OVERLAP_R sets R (default sm_count / 3 + 1).
// The decision itself, on plain arrays (also behind ssdk_schedule_preview, so that it is testable without a device).
// kind[i]: 0 = not a tensor-core GEMM launch (pool, L2Norm, input, image-facing conv), 1 = trunk convolution, 2 = predictor head;
// grid[i]: CTAs of the launch (kind > 0); input[i]: producing layer or -1.  Returns the first side-stream layer (-1: one stream).
int overlap_assign(int n, const int* kind, const int* grid, const int* input, int R, int sm_count, uint8_t* on_side, int* grid_cap) {
  for (int i = 0; i < n; ++i) on_side[i] = 0;
  *grid_cap = 0;
  // first trunk convolution from which on all trunk convolutions are narrow
  int from = -1;
  for (int i = n - 1; i >= 0; --i) {
    if (kind[i] == 2) continue;                 // heads do not decide where the trunk turns narrow
    if (kind[i] == 0) continue;
    if (grid[i] > R) break;
    from = i;
  }
  if (from < 0) return -1;
  int widest = 0, wide_after = 0;
  for (int i = from; i < n; ++i) {
    if (kind[i] > 0) {
      if (grid[i] <= R) { on_side[i] = 1; widest = std::max(widest, grid[i]); }
      else ++wide_after;
    } else if (input[i] >= 0 && on_side[input[i]]) {
      on_side[i] = 1;                           // element-wise consumer of a narrow producer: stays on its producer's stream
    }
  }
  if (!wide_after || !widest) {                 // nothing to run next to the narrow launches
    for (int i = 0; i < n; ++i) on_side[i] = 0;
    return -1;
  }
  *grid_cap = std::max(1, sm_count - widest);
  return from;
}

int plan_overlap(ssdk_model* m) {
  const int n = (int)m->layers.size();
  m->on_side.assign(n, 0);
  m->overlap_from = -1; m->grid_cap = 0;
  if (m->training) return SSDK_OK;
  if (const char* e = getenv("SSDK_OVERLAP")) { if (!atoi(e)) return SSDK_OK; }
  int R = m->ctx->sm_count / 3 + 1;
  if (const char* e = getenv("SSDK_OVERLAP_R")) R = atoi(e);
  std::vector<int> kind(n, 0), grid(n, 0), input(n, -1);
  for (int i = 0; i < n; ++i) {
    const LayerPlan& L = m->layers[i];
    const bool gemm = (L.d.op == SSDK_OP_CONV || L.d.op == SSDK_OP_HEAD) && !L.direct;
    // an image-facing (direct) convolution in the trunk ends the narrow suffix like a wide one: give it a grid no R admits
    if (L.d.op == SSDK_OP_CONV && L.direct) { kind[i] = 1; grid[i] = 1 << 30; }
    else if (gemm) { kind[i] = L.d.op == SSDK_OP_HEAD ? 2 : 1; grid[i] = L.launch.grid; }
    input[i] = (L.d.op == SSDK_OP_INPUT || L.d.op == SSDK_OP_TENSOR) ? -1 : L.d.input;
  }
  m->overlap_from = overlap_assign(n, kind.data(), grid.data(), input.data(), R, m->ctx->sm_count, m->on_side.data(), &m->grid_cap);
  if (m->overlap_from < 0) return SSDK_OK;
  int lo = 0, hi = 0;
  SSDK_CHECK_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
  SSDK_CHECK_CUDA(cudaStreamCreateWithPriority(&m->side, cudaStreamNonBlocking, hi));
  m->dep_ev.resize(n + 1, nullptr);
  for (auto& e : m->dep_ev) SSDK_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  return SSDK_OK;
}

}  // namespace

namespace ssdk {

// One element of the packed planes per thread: row `row`, K index `k` of `layout` <- the master element it holds (or 0)
__global__ void repack_kernel(const float* __restrict__ w, int taps, int cin, int cout, WeightLayout layout, int kblocks, size_t krow,
                              int rows, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)rows * krow) return;
  const int row = (int)(i / krow); const size_t k = i % krow;
  float val = 0.f;
  if (layout == PACK_FWD) {
    const int t = (int)(k / ((size_t)kblocks * 64)), c = (int)(k % ((size_t)kblocks * 64));
    if (t < taps && c < cin) val = w[((size_t)t * cin + c) * cout + row];
  } else if (layout == PACK_FWD_IM2COL) {
    if (k < (size_t)taps * cin) val = w[k * cout + row];
  } else if (layout == PACK_DGRAD) {
    const int t2 = (int)(k / ((size_t)kblocks * 64)), co = (int)(k % ((size_t)kblocks * 64));
    if (t2 < taps && co < cout) val = w[((size_t)(taps - 1 - t2) * cin + row) * cout + co];
  } else {
    if (k < (size_t)cout) val = w[(size_t)row * cout + k];
  }
  split_store(hi, lo, i, val);
}

int launch_repack(ssdk_ctx* ctx, const float* w, int taps, int cin, int cout, WeightLayout layout, int kblocks, size_t krow,
                  __nv_bfloat16* hi, __nv_bfloat16* lo, cudaStream_t s) {
  const int rows = layout == PACK_DGRAD ? cin : layout == PACK_DGRAD_COL ? taps * cin : cout;
  const size_t total = (size_t)rows * krow;
  repack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(w, taps, cin, cout, layout, kblocks, krow, rows, hi, lo);
  SSDK_COUNT_LAUNCH(ctx);
  SSDK_CHECK_CUDA(cudaGetLastError());
  return SSDK_OK;
}

// Geometry, tile list, pipeline depths and TMA descriptors of one implicit-GEMM launch.  The caller fills the epilogue.
int plan_conv_gemm(ssdk_model* m, ConvLaunch& cl, const ConvGeom& g, const __nv_bfloat16* w_hi, const __nv_bfloat16* w_lo,
                   size_t krow, int kblocks, int** tile_list_out) {
  ConvArgs& a = cl.args;
  memset(&a, 0, sizeof(a));
  const __nv_bfloat16* a_hi; const __nv_bfloat16* a_lo;
  uint64_t a_inner, a_rows;
  if (!g.in) {
    SSDK_REQUIRE(g.a_rows < (1ull << 31), "GEMM with too many rows");
    a.M_total = (int)g.a_rows; a.rows_per_img = g.Ho * g.Wo; a.in_Wp = g.Wo;
    a.KH = 1; a.KW = 1; a.row_shift[0] = 0; a.kw_rows = 1;
    a_hi = g.a_hi; a_lo = g.a_lo; a_inner = g.a_inner; a_rows = g.a_rows;
  } else {
    const ActBuf& ia = *g.in;
    SSDK_REQUIRE((long long)g.B * ia.Hp() * ia.Wp() < (1ll << 31), "activation tensor with too many rows");
    a.M_total = g.B * ia.Hp() * ia.Wp(); a.rows_per_img = ia.Hp() * ia.Wp(); a.in_Wp = ia.Wp();
    SSDK_REQUIRE(g.kh <= 8 && g.kw <= 8, "conv kernel %dx%d is larger than the supported 8x8", g.kh, g.kw);
    a.KH = g.kh; a.KW = g.kw; a.kw_rows = g.dilation;
    for (int kh = 0; kh < g.kh; ++kh) {
      a.row_shift[kh] = (kh * g.dilation - g.pad_t + ia.pad) * ia.Wp() + (0 - g.pad_l + ia.pad);
      SSDK_REQUIRE(a.row_shift[kh] >= 0, "internal: activation border too small for this convolution");
    }
    a_hi = ia.hi; a_lo = ia.lo; a_inner = ia.Cs; a_rows = (uint64_t)a.M_total;
  }
  a.kblocks = kblocks;
  a.Ho = g.Ho; a.Wo = g.Wo; a.B = g.B;
  a.cout = g.cout;
  a.BN = g.cout <= 64 ? 64 : (g.cout <= 128 ? 128 : 256);
  a.split = m->split;
  a.k_split = 1;
  if (a.split && a.BN == 256) {
    // bf16x3 tiles carry the cross-term accumulator (acc_split), which fits in registers up to 160 columns: 160-wide tiles for
    // the predictor heads of <= 160 columns (6 boxes x 25 for VOC: the fused head epilogue needs all boxes of a pixel in one
    // tile), 128-wide tiles otherwise
    a.BN = g.cout <= 160 ? 160 : 128;
  } else if (a.BN == 256 && g.cout % 128 == 0) {                // (not the predictor heads: their epilogue needs all boxes in one tile)
    // 256-wide tiles on few m-tiles leave the last wave of the persistent grid mostly empty; 128-wide tiles double the units.
    // Pick the width with fewer tile-columns per SM over all waves (a partial last wave costs a whole one).
    long long n_valid = 0;
    for (long long t = 0; t < (a.M_total + 127) / 128; ++t) {
      bool any = false;
      for (int r = 0; r < 128 && !any; ++r) {
        const long long v = t * 128 + r;
        if (v >= a.M_total) break;
        const int rr = (int)(v % a.rows_per_img);
        any = (rr / a.in_Wp < g.Ho) && (rr % a.in_Wp < g.Wo);
      }
      n_valid += any;
    }
    const int sms = m->ctx->sm_count;
    const long long u256 = n_valid * ((g.cout + 255) / 256), u128 = n_valid * ((g.cout + 127) / 128);
    const double t256 = (double)((u256 + sms - 1) / sms) * 256.0;
    const double t128 = (double)((u128 + sms - 1) / sms) * 128.0;
    const bool use128 = t128 < t256;
    if (use128) a.BN = 128;
  }
  a.acc_split = a.split;
  a.n_tiles_n = (g.cout + a.BN - 1) / a.BN;
  const int n_m = (a.M_total + 127) / 128;
  conv_pick_stages(a);
  // m-tiles that hold at least one valid output row
  std::vector<int> tiles;
  for (int t = 0; t < n_m; ++t) {
    bool any = false;
    for (int r = 0; r < 128 && !any; ++r) {
      long long v = (long long)t * 128 + r;
      if (v >= a.M_total) break;
      int rr = (int)(v % a.rows_per_img);
      any = (rr / a.in_Wp < g.Ho) && (rr % a.in_Wp < g.Wo);
    }
    if (any) tiles.push_back(t);
  }
  a.n_tiles_m = (int)tiles.size();
  int* tl = nullptr;
  int rc = dev_alloc(m->allocs, &tl, tiles.size(), false); if (rc) return rc;
  SSDK_CHECK_CUDA(cudaMemcpy(tl, tiles.data(), tiles.size() * sizeof(int), cudaMemcpyHostToDevice));
  a.tile_list = tl;
  if (tile_list_out) *tile_list_out = tl;
  const uint64_t a_ld = (!g.in && g.a_ld) ? g.a_ld : a_inner;
  rc = make_tmap_2d(&cl.a_hi, a_hi, a_inner, a_rows, a_ld * 2, 64, 128); if (rc) return rc;
  rc = make_tmap_2d(&cl.b_hi, w_hi, krow, (uint64_t)g.cout, krow * 2, 64, (uint32_t)a.BN); if (rc) return rc;
  if (m->split) {
    rc = make_tmap_2d(&cl.a_lo, a_lo, a_inner, a_rows, a_ld * 2, 64, 128); if (rc) return rc;
    rc = make_tmap_2d(&cl.b_lo, w_lo, krow, (uint64_t)g.cout, krow * 2, 64, (uint32_t)a.BN); if (rc) return rc;
  } else { cl.a_lo = cl.a_hi; cl.b_lo = cl.b_hi; }
  const int total_tiles = a.n_tiles_m * a.n_tiles_n;
  cl.grid = std::max(1, std::min(total_tiles, m->ctx->sm_count));
  cl.smem = conv_smem_bytes(a);
  SSDK_REQUIRE(cl.smem <= 227 * 1024, "internal: conv plan needs %zu bytes of shared memory", cl.smem);
  double issued = 0;
  for (int nt = 0; nt < a.n_tiles_n; ++nt) {
    // every tile issues the full BN columns (the weight rows past cout are TMA zero fill) and all 64 channels of every k-block,
    // 3 products with split planes
    issued += 2.0 * a.n_tiles_m * 128.0 * a.BN * (m->split ? 3.0 : 1.0) * (double)(a.KH * a.KW) * (kblocks * 64);
  }
  cl.flops_issued = issued;
  return SSDK_OK;
}

}  // namespace ssdk

extern "C" int ssdk_model_create(ssdk_ctx* ctx, const ssdk_model_desc* desc, ssdk_model** out) {
  SSDK_REQUIRE(ctx && desc && out && desc->layers && desc->n_layers > 0, "ssdk_model_create: bad argument");
  SSDK_REQUIRE(desc->batch > 0 && desc->img_height > 0 && desc->img_width > 0, "ssdk_model_create: bad input shape");
  SSDK_REQUIRE(desc->precision == 0 || desc->precision == 1, "ssdk_model_create: precision must be 0 (bf16x3) or 1 (bf16)");
  SSDK_REQUIRE(ctx->prop.major == 9 && ctx->prop.minor == 0,
               "libssdk's convolution kernels need an sm_90 (Hopper) GPU, found sm_%d%d; there is no fallback", ctx->prop.major, ctx->prop.minor);
  SSDK_CHECK_CUDA(cudaSetDevice(ctx->device));
  ssdk_model* m = new ssdk_model();
  m->ctx = ctx; m->B = desc->batch; m->H = desc->img_height; m->W = desc->img_width; m->Cimg = desc->img_channels;
  m->Ctot = desc->n_classes_total; m->split = desc->precision == 0 ? 1 : 0; m->training = desc->training ? 1 : 0;
  for (int i = 0; i < 4; ++i) m->var[i] = desc->variances[i];
  const int n = desc->n_layers;
  m->layers.resize(n);
  int rc = SSDK_OK;
  auto fail = [&](int code) { ssdk_model_destroy(m); return code; };
  // pass 1: shapes
  for (int i = 0; i < n; ++i) {
    LayerPlan& L = m->layers[i];
    L.d = desc->layers[i];
    const ssdk_layer_desc& d = L.d;
    if (d.op == SSDK_OP_TENSOR) { L.H = m->H; L.W = m->W; L.C = m->Cimg; continue; }
    if (d.op == SSDK_OP_INPUT) {
      L.H = m->H; L.W = m->W; L.C = m->Cimg;
      if (d.mean) { L.has_mean = true; for (int c = 0; c < 3; ++c) L.mean[c] = d.mean[c]; }
      if (d.stddev) { L.has_std = true; for (int c = 0; c < 3; ++c) L.stddev[c] = d.stddev[c]; }
      if (d.swap) { L.has_swap = true; for (int c = 0; c < 3; ++c) L.swap[c] = d.swap[c]; }
      continue;
    }
    if (!(d.input >= 0 && d.input < i)) { set_error("layer %d: input %d must refer to an earlier layer", i, d.input); return fail(SSDK_ERR_INVALID); }
    const LayerPlan& in = m->layers[d.input];
    if (in.d.op == SSDK_OP_HEAD) { set_error("layer %d: a head cannot feed another layer", i); return fail(SSDK_ERR_INVALID); }
    L.in_H = in.H; L.in_W = in.W; L.in_C = in.C;
    if (d.op == SSDK_OP_CONV || d.op == SSDK_OP_HEAD) {
      if (d.kh <= 0 || d.kw <= 0 || d.stride <= 0 || d.dilation <= 0) { set_error("layer %d: bad conv geometry", i); return fail(SSDK_ERR_INVALID); }
      L.H = (in.H + d.pad_t + d.pad_b - d.dilation * (d.kh - 1) - 1) / d.stride + 1;
      L.W = (in.W + d.pad_l + d.pad_r - d.dilation * (d.kw - 1) - 1) / d.stride + 1;
      L.C = d.op == SSDK_OP_HEAD ? d.n_boxes * (m->Ctot + 4) : d.cout;
      if (L.H <= 0 || L.W <= 0 || L.C <= 0) { set_error("layer %d: empty conv output", i); return fail(SSDK_ERR_INVALID); }
    } else if (d.op == SSDK_OP_MAXPOOL) {
      L.H = (in.H + d.pad_t + d.pad_b - d.kh) / d.stride + 1;
      L.W = (in.W + d.pad_l + d.pad_r - d.kw) / d.stride + 1;
      L.C = in.C;
    } else if (d.op == SSDK_OP_L2NORM) {
      L.H = in.H; L.W = in.W; L.C = in.C;
    } else { set_error("layer %d: unknown op %d", i, d.op); return fail(SSDK_ERR_INVALID); }
  }
  // pass 2: border each producer must provide (max over its virtual-path conv consumers)
  for (int i = 0; i < n; ++i) {
    const ssdk_layer_desc& d = m->layers[i].d;
    if (d.op != SSDK_OP_CONV && d.op != SSDK_OP_HEAD) continue;
    LayerPlan& in = m->layers[d.input];
    const bool im2col = (d.stride != 1) || (in.C < 8);
    if (!im2col) in.need_pad = std::max(in.need_pad, std::max(std::max(d.pad_t, d.pad_b), std::max(d.pad_l, d.pad_r)));
    // the image-facing layer's gathered A tile (conv_first_kernel) reads its taps from the input planes' zero border
    if (!desc->training && in.C < 8 && d.stride == 1)
      in.need_pad = std::max(in.need_pad, std::max(std::max(d.pad_t, d.pad_l),
                                                   std::max((d.kh - 1) * d.dilation - d.pad_t, (d.kw - 1) * d.dilation - d.pad_l)));
    // training: the image-facing weight-gradient kernel reads its 3x3 window without bounds checks
    if (desc->training && in.C < 8 && d.stride == 1)
      in.need_pad = std::max(in.need_pad, d.dilation * std::max(d.kh - 1, d.kw - 1));
    if (desc->training && !im2col) {
      // the gradient of this layer's output shares the geometry of the output itself and is the input of the
      // data-gradient convolution, whose padding is dilation*(k-1) - pad
      LayerPlan& self = m->layers[i];
      const int pt = d.dilation * (d.kh - 1) - d.pad_t, pb = d.dilation * (d.kh - 1) - d.pad_b;
      const int pl = d.dilation * (d.kw - 1) - d.pad_l, pr = d.dilation * (d.kw - 1) - d.pad_r;
      self.need_pad = std::max(self.need_pad, std::max(std::max(pt, pb), std::max(pl, pr)));
    }
  }
  // pass 3: buffers, weights, launches
  rc = tma_init(); if (rc) return fail(rc);
  int prior_off = 0;
  for (int i = 0; i < n; ++i) {
    LayerPlan& L = m->layers[i];
    const ssdk_layer_desc& d = L.d;
    if (d.op != SSDK_OP_HEAD) { rc = alloc_act(m, L.out, m->B, L.H, L.W, L.C, L.need_pad); if (rc) return fail(rc); }
    if (d.op == SSDK_OP_CONV || d.op == SSDK_OP_HEAD) {
      if (!d.kernel || (d.op == SSDK_OP_HEAD && !d.kernel2)) { set_error("layer %d: missing kernel", i); return fail(SSDK_ERR_INVALID); }
      rc = build_conv(m, i); if (rc) return fail(rc);
      if (d.op == SSDK_OP_HEAD) { L.prior_off = prior_off; prior_off += L.H * L.W * d.n_boxes; }
      cudaEventCreate(&L.ev0); cudaEventCreate(&L.ev1);
    } else if (d.op == SSDK_OP_L2NORM) {
      if (!d.kernel) { set_error("layer %d: L2Normalization needs gamma in `kernel`", i); return fail(SSDK_ERR_INVALID); }
      rc = upload_f32(m, &L.gamma, d.kernel, L.C); if (rc) return fail(rc);
    }
  }
  m->P = prior_off;
  if (m->P > 0) {
    if (!desc->anchors_f32) { set_error("ssdk_model_create: anchors_f32 is NULL"); return fail(SSDK_ERR_INVALID); }
    rc = upload_f32(m, &m->d_anchors, desc->anchors_f32, (size_t)m->P * 4); if (rc) return fail(rc);
  }
  for (auto& L : m->layers)
    if (L.head_fused) {
      ConvArgs& a = L.launch.args;
      a.head_P = m->P; a.head_prior_off = L.prior_off; a.head_anchors = m->d_anchors;
      for (int k = 0; k < 4; ++k) a.head_var[k] = m->var[k];
    }
  rc = plan_overlap(m); if (rc) return fail(rc);
  SSDK_CHECK_CUDA(cudaDeviceSynchronize());
  *out = m;
  return SSDK_OK;
}

extern "C" int ssdk_model_destroy(ssdk_model* m) {
  if (!m) return SSDK_OK;
  for (auto& L : m->layers) { if (L.ev0) cudaEventDestroy(L.ev0); if (L.ev1) cudaEventDestroy(L.ev1); }
  for (auto& e : m->dep_ev) if (e) cudaEventDestroy(e);
  if (m->side) { cudaStreamSynchronize(m->side); cudaStreamDestroy(m->side); }
  for (void* p : m->allocs) cudaFree(p);
  delete m;
  return SSDK_OK;
}

extern "C" int ssdk_model_num_priors(const ssdk_model* m, int* out_P) {
  SSDK_REQUIRE(m && out_P, "ssdk_model_num_priors: NULL argument");
  *out_P = m->P;
  return SSDK_OK;
}

extern "C" int ssdk_model_layer_shape(const ssdk_model* m, int layer, int* h, int* w, int* c) {
  SSDK_REQUIRE(m && layer >= 0 && layer < (int)m->layers.size(), "ssdk_model_layer_shape: bad layer index");
  if (h) *h = m->layers[layer].H;
  if (w) *w = m->layers[layer].W;
  if (c) *c = m->layers[layer].C;
  return SSDK_OK;
}

extern "C" int ssdk_model_layer_plan(const ssdk_model* m, int layer, ssdk_layer_plan* out) {
  SSDK_REQUIRE(m && out && layer >= 0 && layer < (int)m->layers.size(), "ssdk_model_layer_plan: bad argument");
  memset(out, 0, sizeof(*out));
  const LayerPlan& L = m->layers[layer];
  if (L.d.op != SSDK_OP_CONV && L.d.op != SSDK_OP_HEAD) return SSDK_OK;
  out->split = m->split;
  if (L.direct && L.first_tc) {
    out->kernel = SSDK_PLAN_FIRST_TC;
    out->bn = L.first.BN; out->kblocks = L.first.kblocks;
    out->n_tiles_m = L.first.n_tiles; out->n_tiles_n = 1;
    out->grid = L.first.grid; out->k_split = 1;
    return SSDK_OK;
  }
  if (L.direct) { out->kernel = SSDK_PLAN_DIRECT; out->split = 0; return SSDK_OK; }
  const ConvArgs& a = L.launch.args;
  out->kernel = L.im2col ? SSDK_PLAN_IM2COL_GEMM : SSDK_PLAN_GEMM;
  out->bn = a.BN; out->split = a.split; out->stages = a.stages; out->kblocks = a.kblocks;
  out->n_tiles_m = a.n_tiles_m; out->n_tiles_n = a.n_tiles_n; out->grid = L.launch.grid; out->k_split = a.k_split > 1 ? a.k_split : 1;
  out->epilogue = a.epi; out->head_fused = L.head_fused ? 1 : 0;
  out->im2col_vec8 = L.im2col && L.im2col_vec8 ? 1 : 0;
  return SSDK_OK;
}

extern "C" int ssdk_model_flops(const ssdk_model* m, double* algo, double* issued) {
  SSDK_REQUIRE(m, "ssdk_model_flops: NULL model");
  if (algo) *algo = m->flops_algo;
  if (issued) *issued = m->flops_issued;
  return SSDK_OK;
}

extern "C" int ssdk_model_set_timing(ssdk_model* m, int enable) {
  SSDK_REQUIRE(m, "ssdk_model_set_timing: NULL model");
  m->timing = enable ? 1 : 0;
  return SSDK_OK;
}

extern "C" int ssdk_model_last_conv_ms(ssdk_model* m, float* out_ms) {
  SSDK_REQUIRE(m && out_ms, "ssdk_model_last_conv_ms: NULL argument");
  float total = 0.f;
  for (auto& L : m->layers) {
    if (!L.ev0 || L.direct) continue;
    SSDK_CHECK_CUDA(cudaEventSynchronize(L.ev1));
    float ms = 0.f;
    SSDK_CHECK_CUDA(cudaEventElapsedTime(&ms, L.ev0, L.ev1));
    total += ms;
  }
  *out_ms = total;
  return SSDK_OK;
}

extern "C" int ssdk_model_layer_ms(const ssdk_model* m, int layer, float* out_ms) {
  SSDK_REQUIRE(m && out_ms && layer >= 0 && layer < (int)m->layers.size(), "ssdk_model_layer_ms: bad argument");
  const LayerPlan& L = m->layers[layer];
  *out_ms = 0.f;
  if (!L.ev0 || L.direct) return SSDK_OK;
  SSDK_CHECK_CUDA(cudaEventSynchronize(L.ev1));
  SSDK_CHECK_CUDA(cudaEventElapsedTime(out_ms, L.ev0, L.ev1));
  return SSDK_OK;
}

extern "C" int ssdk_model_forward(ssdk_model* m, const float* images_dev, float* y_pred_dev, void* stream_) {
  SSDK_REQUIRE(m && images_dev, "ssdk_model_forward: NULL argument");
  SSDK_REQUIRE(m->P == 0 || y_pred_dev, "ssdk_model_forward: y_pred_dev is NULL");
  cudaStream_t main_stream = (cudaStream_t)stream_;
  ssdk_ctx* ctx = m->ctx;
  int rc;
  // two-stream schedule (plan_overlap); instrumented passes (per-launch events) stay on one stream
  const bool overlap = m->overlap_from >= 0 && !m->timing;
  // issue counters per stream (0: caller's, 1: side) and, per consumer stream, how much of the OTHER stream it has already waited for
  int issued[2] = {0, 0}, seen[2] = {0, 0}, side_used = 0;
  std::vector<int>& pos = m->issue_pos;
  pos.assign(m->layers.size(), 0);
  for (size_t i = 0; i < m->layers.size(); ++i) {
    LayerPlan& L = m->layers[i];
    const ssdk_layer_desc& d = L.d;
    const int sx = overlap && m->on_side[i] ? 1 : 0;
    cudaStream_t stream = sx ? m->side : main_stream;
    int cap = 0;
    if (overlap) {
      if (d.op != SSDK_OP_INPUT && d.input >= 0) {
        const int sy = m->on_side[d.input] ? 1 : 0;
        // the first launch on the side stream also orders it behind everything the caller's stream holds (previous calls included)
        const bool first_side = sx == 1 && !side_used;
        if ((sy != sx && pos[d.input] > seen[sx]) || first_side) {
          cudaStream_t other = sx ? main_stream : m->side;
          SSDK_CHECK_CUDA(cudaEventRecord(m->dep_ev[i], other));
          SSDK_CHECK_CUDA(cudaStreamWaitEvent(stream, m->dep_ev[i], 0));
          seen[sx] = issued[sx ^ 1];
        }
      }
      if (sx) side_used = 1;
      pos[i] = ++issued[sx];
      if (!sx && side_used) cap = m->grid_cap;
    }
    switch (d.op) {
      case SSDK_OP_TENSOR:
        rc = launch_pack(ctx, images_dev, L.out, stream);
        if (rc) return rc;
        break;
      case SSDK_OP_INPUT:
        rc = launch_preprocess(ctx, images_dev, m->B, m->H, m->W, m->Cimg, L.has_mean ? L.mean : nullptr,
                               L.has_std ? L.stddev : nullptr, L.has_swap ? L.swap : nullptr, L.out, stream);
        if (rc) return rc;
        break;
      case SSDK_OP_CONV:
      case SSDK_OP_HEAD: {
        const LayerPlan& in = m->layers[d.input];
        if (L.direct) {
          if (L.first_tc)
            rc = launch_conv_first(ctx, L.first, in.out, L.out, L.w_hi, L.w_lo, L.bias, L.bn_scale, L.bn_shift, d.act, d.kh, d.kw, d.dilation, d.pad_t,
                                   d.pad_l, stream);
          else
          rc = launch_conv_direct(ctx, in.out, L.bn_train ? L.z : L.out, L.w_f32, L.bias, L.bn_scale, L.bn_shift, L.bn_train ? (int)SSDK_ACT_NONE : d.act,
                                  d.kh, d.kw, d.dilation, d.pad_t, d.pad_l, stream);
          if (rc) return rc;
          if (L.bn_train) { rc = launch_bn_forward(ctx, L, d.act, stream); if (rc) return rc; }
          break;
        }
        if (L.im2col) {
          rc = launch_im2col(ctx, in.out, L.col_hi, L.col_lo, L.H, L.W, d.kh, d.kw, d.stride, d.dilation, d.pad_t, d.pad_l, L.Kpad, L.im2col_vec8, stream);
          if (rc) return rc;
        }
        if (m->timing) cudaEventRecord(L.ev0, stream);
        if (L.head_fused) L.launch.args.out_f32 = y_pred_dev;                   // the epilogue writes the prediction rows themselves
        rc = launch_conv(ctx, L.launch, stream, cap);
        if (rc) return rc;
        if (m->timing) cudaEventRecord(L.ev1, stream);
        if (L.bn_train) { rc = launch_bn_forward(ctx, L, d.act, stream); if (rc) return rc; }
        if (d.op == SSDK_OP_HEAD && !L.head_fused) {
          rc = launch_head_finalize(ctx, L.head_f32, m->B, L.H * L.W, d.n_boxes, m->Ctot, m->P, L.prior_off, m->d_anchors, m->var,
                                    y_pred_dev, stream);
          if (rc) return rc;
        }
        break;
      }
      case SSDK_OP_MAXPOOL:
        rc = launch_maxpool(ctx, m->layers[d.input].out, L.out, d.kh, d.kw, d.stride, d.pad_t, d.pad_l, stream);
        if (rc) return rc;
        break;
      case SSDK_OP_L2NORM:
        rc = launch_l2norm(ctx, m->layers[d.input].out, L.out, L.gamma, stream);
        if (rc) return rc;
        break;
      default:
        break;
    }
  }
  if (side_used) {                             // join: whatever the caller enqueues next sees the finished prediction tensor
    SSDK_CHECK_CUDA(cudaEventRecord(m->dep_ev.back(), m->side));
    SSDK_CHECK_CUDA(cudaStreamWaitEvent(main_stream, m->dep_ev.back(), 0));
  }
  return SSDK_OK;
}

extern "C" int ssdk_model_read_layer(ssdk_model* m, int layer, float* out_dev, void* stream_) {
  SSDK_REQUIRE(m && out_dev && layer >= 0 && layer < (int)m->layers.size(), "ssdk_model_read_layer: bad argument");
  LayerPlan& L = m->layers[layer];
  cudaStream_t stream = (cudaStream_t)stream_;
  if (L.d.op == SSDK_OP_HEAD) {
    SSDK_REQUIRE(L.head_f32, "ssdk_model_read_layer: this plan writes the predictor outputs straight into y_pred (no separate head tensor)");
    SSDK_CHECK_CUDA(cudaMemcpyAsync(out_dev, L.head_f32, (size_t)m->B * L.H * L.W * L.C * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    return SSDK_OK;
  }
  return launch_unpack(m->ctx, L.out, out_dev, stream);
}

extern "C" int ssdk_model_layer_planes_shape(const ssdk_model* m, int layer, int* out_hp, int* out_wp, int* out_cs, int* out_pad) {
  SSDK_REQUIRE(m && out_hp && out_wp && out_cs && out_pad && layer >= 0 && layer < (int)m->layers.size(), "ssdk_model_layer_planes_shape: bad argument");
  const ActBuf& o = m->layers[layer].out;
  SSDK_REQUIRE(o.hi, "ssdk_model_layer_planes_shape: layer %d has no activation planes", layer);
  *out_hp = o.Hp(); *out_wp = o.Wp(); *out_cs = o.Cs; *out_pad = o.pad;
  return SSDK_OK;
}

extern "C" int ssdk_model_read_layer_planes(ssdk_model* m, int layer, uint16_t* hi_dev, uint16_t* lo_dev, void* stream) {
  SSDK_REQUIRE(m && hi_dev && layer >= 0 && layer < (int)m->layers.size(), "ssdk_model_read_layer_planes: bad argument");
  const ActBuf& o = m->layers[layer].out;
  SSDK_REQUIRE(o.hi, "ssdk_model_read_layer_planes: layer %d has no activation planes", layer);
  const size_t bytes = o.elems() * sizeof(uint16_t);
  SSDK_CHECK_CUDA(cudaMemcpyAsync(hi_dev, o.hi, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  if (lo_dev && o.lo) SSDK_CHECK_CUDA(cudaMemcpyAsync(lo_dev, o.lo, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return SSDK_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Stand-alone layer calls (SURVEY 8b: ssdk_conv2d_fwd, ssdk_maxpool): a one-layer graph through the same plan builder
// ---------------------------------------------------------------------------------------------------------------------
namespace {
int run_single_layer(ssdk_ctx* ctx, const float* x_dev, int B, int H, int W, int C, const ssdk_layer_desc& layer, int precision,
                     float* y_dev, void* stream) {
  ssdk_layer_desc layers[2];
  memset(layers, 0, sizeof(layers));
  layers[0].op = SSDK_OP_TENSOR; layers[0].input = -1;
  layers[1] = layer; layers[1].input = 0;
  ssdk_model_desc md;
  memset(&md, 0, sizeof(md));
  md.batch = B; md.img_height = H; md.img_width = W; md.img_channels = C; md.n_classes_total = 0;
  md.n_layers = 2; md.layers = layers; md.precision = precision; md.anchors_f32 = nullptr; md.training = 0;
  ssdk_model* m = nullptr;
  int rc = ssdk_model_create(ctx, &md, &m);
  if (rc) return rc;
  rc = ssdk_model_forward(m, x_dev, nullptr, stream);
  if (!rc) rc = ssdk_model_read_layer(m, 1, y_dev, stream);
  const cudaError_t e = cudaStreamSynchronize((cudaStream_t)stream);     // the plan's buffers are freed below
  ssdk_model_destroy(m);
  if (!rc && e != cudaSuccess) { set_error("ssdk single-layer call failed: %s", cudaGetErrorString(e)); return SSDK_ERR_CUDA; }
  return rc;
}
}  // namespace

extern "C" int ssdk_conv2d_fwd(ssdk_ctx* ctx, const float* x_dev, int B, int H, int W, int Cin, const float* kernel_hwio_host,
                               const float* bias_host, int Cout, int kh, int kw, int stride, int dilation, int pad_t, int pad_l,
                               int pad_b, int pad_r, int act, int precision, float* y_dev, void* stream) {
  SSDK_REQUIRE(ctx && x_dev && kernel_hwio_host && y_dev, "ssdk_conv2d_fwd: NULL argument");
  SSDK_REQUIRE(B > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "ssdk_conv2d_fwd: bad tensor shape");
  SSDK_REQUIRE(Cout % 8 == 0, "ssdk_conv2d_fwd: output channels must be a multiple of 8 (got %d)", Cout);
  SSDK_REQUIRE(Cin >= 8 || (stride == 1 && Cin <= 4), "ssdk_conv2d_fwd: 5..7 input channels are not supported (pad the tensor to 8)");
  SSDK_REQUIRE(pad_t >= 0 && pad_l >= 0 && pad_b >= 0 && pad_r >= 0, "ssdk_conv2d_fwd: negative padding");
  ssdk_layer_desc d;
  memset(&d, 0, sizeof(d));
  std::vector<float> zero_bias;
  if (!bias_host) { zero_bias.assign(Cout, 0.f); bias_host = zero_bias.data(); }
  d.op = SSDK_OP_CONV; d.cout = Cout; d.kh = kh; d.kw = kw; d.stride = stride; d.dilation = dilation;
  d.pad_t = pad_t; d.pad_l = pad_l; d.pad_b = pad_b; d.pad_r = pad_r; d.act = act;
  d.kernel = kernel_hwio_host; d.bias = bias_host;
  return run_single_layer(ctx, x_dev, B, H, W, Cin, d, precision, y_dev, stream);
}

extern "C" int ssdk_maxpool(ssdk_ctx* ctx, const float* x_dev, int B, int H, int W, int C, int kh, int kw, int stride, int pad_t,
                            int pad_l, int pad_b, int pad_r, float* y_dev, void* stream) {
  SSDK_REQUIRE(ctx && x_dev && y_dev, "ssdk_maxpool: NULL argument");
  SSDK_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && kh > 0 && kw > 0 && stride > 0, "ssdk_maxpool: bad argument");
  SSDK_REQUIRE(pad_t >= 0 && pad_l >= 0 && pad_b >= 0 && pad_r >= 0 && pad_t < kh && pad_l < kw, "ssdk_maxpool: bad padding");
  ssdk_layer_desc d;
  memset(&d, 0, sizeof(d));
  d.op = SSDK_OP_MAXPOOL; d.kh = kh; d.kw = kw; d.stride = stride; d.dilation = 1;
  d.pad_t = pad_t; d.pad_l = pad_l; d.pad_b = pad_b; d.pad_r = pad_r;
  return run_single_layer(ctx, x_dev, B, H, W, C, d, 0, y_dev, stream);
}

extern "C" int ssdk_schedule_preview(int n_layers, const int* kind, const int* grid, const int* input, int R, int sm_count,
                                     unsigned char* out_on_side, int* out_from, int* out_grid_cap) {
  SSDK_REQUIRE(n_layers > 0 && kind && grid && input && out_on_side && out_from && out_grid_cap, "ssdk_schedule_preview: bad argument");
  for (int i = 0; i < n_layers; ++i)
    SSDK_REQUIRE(input[i] < i && kind[i] >= 0 && kind[i] <= 2, "ssdk_schedule_preview: layer %d: input must refer to an earlier layer, kind must be 0..2", i);
  *out_from = overlap_assign(n_layers, kind, grid, input, R > 0 ? R : sm_count / 3 + 1, sm_count, out_on_side, out_grid_cap);
  return SSDK_OK;
}
