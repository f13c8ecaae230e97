// MO-CMA-ES with its parent state resident in HBM, one generation of MOASMO.optimize's surrogate epoch in two calls.
//   dmo_cmaes_step_record   generate_strategy (dmosopt/CMAES.py:231-271), the surrogate's posterior mean of the offspring
//                           and _select (CMAES.py:167-229): everything up to the chosen / not-chosen split of the candidates
//   dmo_cmaes_step_apply    the device half of update_strategy (CMAES.py:273-414): the chosen offspring's strategy
//                           parameters, the parents' step sizes and the next parent set
// Between the two the host runs update_strategy's scalar arithmetic (success rates and NumPy's exp of the step-size
// factors, CMAES._strategy_scalars), which has to be NumPy's to keep the plugin's bits.  The normal variates and the parent
// draws are the caller's (local_random), drawn before the first call.  Both calls are compositions of the device bodies
// of dmo_rank_nd, dmo_cmaes_generate, the predict, dmo_ehvi_select, dmo_gather_rows, dmo_scale_rows, dmo_cmaes_step_z and
// dmo_cmaes_update_cholesky; the new kernels below cut the fronts, draw the parents and assemble the next parent set.
// None of them runs beside a GP variance contraction (no lane is forked here); each is one pass per element with
// atomics at most, so none needs its CTAs resident together.
#include "common.cuh"
#include "gp.cuh"

namespace {

// p_idx[i] = order[js[i]]: the parents drawn among the first entries of the stable rank order (CMAES.py:249-262)
__global__ void cmaes_pick_parents_kernel(const uint32_t* __restrict__ order, const int64_t* __restrict__ js, int64_t n,
                                          int64_t* __restrict__ p_idx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p_idx[i] = (int64_t)order[js[i]];
}

// counts[r] = rows of rank r (ranks in [0, n))
__global__ void rank_hist_kernel(const int32_t* __restrict__ rank, int64_t n, int32_t* __restrict__ counts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(&counts[rank[i]], 1);
}

// b = cumulative front sizes (b[0] = 0, b[n] = n).  _select maps its fronts through the inverse of the stable rank order
// (CMAES.py:190), so "front r" is the candidate rows [b[r], b[r + 1]) in candidate order.  Whole fronts are chosen while
// they fit in pop; the front R with b[R] <= pop < b[R + 1] is the mid front: cut = (b[R], b[R + 1]).  Exactly one R
// exists, since b[0] = 0 <= pop < n = b[n].
__global__ void front_cut_kernel(const int32_t* __restrict__ b, int64_t n, int64_t pop, int64_t* __restrict__ cut) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
    if ((int64_t)b[r] <= pop && (int64_t)b[r + 1] > pop) {
      cut[0] = b[r];
      cut[1] = b[r + 1];
    }
}

// code[i] = 1 for the rows of the whole fronts chosen (i < cut[0]), 0 for the others; the mid front's picks follow
__global__ void front_codes_kernel(const int64_t* __restrict__ cut, int64_t n, uint8_t* __restrict__ code) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) code[i] = i < cut[0] ? 1 : 0;
}

// the k picks of the mid front: rows cut[0] + sel[j] (the hypervolume-improvement selection) or cut[0] + j when nothing
// was chosen before it (sel == nullptr: np.arange(k), CMAES.py:207-210)
__global__ void mid_pick_kernel(const int64_t* __restrict__ cut, const int64_t* __restrict__ sel, int64_t k, uint8_t* __restrict__ code) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < k) code[cut[0] + (sel ? sel[j] : j)] = 1;
}

// ref[j] = max(Y[:, j]) + 1 (CMAES.py:203): NaN propagates as in np.max; in float32 arithmetic when the candidates are a
// float32 array (one rounding of the float32 sum, as NumPy adds)
constexpr int kMaxT = 256;
__global__ void __launch_bounds__(kMaxT) ref_point_kernel(const double* __restrict__ Y, int64_t n, int M, int f32, double* __restrict__ ref) {
  __shared__ double red[kMaxT];
  const int j = blockIdx.x;
  double m = -INFINITY;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = Y[i * M + j];
    m = (isnan(m) || v <= m) ? m : v;
  }
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = kMaxT / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      const double a = red[threadIdx.x], c = red[threadIdx.x + s];
      red[threadIdx.x] = (isnan(a) || c <= a) ? a : c;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) ref[j] = f32 ? (double)__fadd_rn((float)red[0], 1.0f) : __dadd_rn(red[0], 1.0);
}

__global__ void fill_kernel(double* __restrict__ a, int64_t n, double v) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

// The next parent set in one pass (CMAES.py:385-411).  Row i comes from candidate ch = cand[i]: an offspring (ch < C)
// brings its row of x_gen and its own updated strategy rows off_*[src[i]]; a surviving parent keeps its rows (parents_x
// row ch - C, strategy rows src[i]).  parents_y and rank are the candidates' rows ch.  Each thread copies one element of
// the row's d + sc + 2 d^2 + d + M + 1 values.
struct Assembly {
  const double *px, *sig, *A, *Ainv, *pc;          // the current parent set
  const double *osig, *oA, *oAinv, *opc;           // the chosen offspring's strategy rows
  const double *cx, *cy;                           // candidates: x_gen (C rows), [y_gen; parents_y]
  const int32_t* crank;                            // candidates' ranks
  const int64_t *cand, *src;                       // (P,) per new row
  double *px_o, *sig_o, *A_o, *Ainv_o, *pc_o, *py_o;
  int32_t* rank_o;
};
__global__ void cmaes_assemble_kernel(Assembly a, int64_t P, int64_t C, int d, int sc, int M) {
  const int64_t dd = (int64_t)d * d;
  const int64_t W = d + sc + 2 * dd + d + M + 1;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= P * W) return;
  const int64_t i = t / W;
  int64_t e = t - i * W;
  const int64_t ch = a.cand[i], s = a.src[i];
  const bool off = ch < C;
  if (e < d) {
    a.px_o[i * d + e] = off ? a.cx[ch * d + e] : a.px[(ch - C) * d + e];
    return;
  }
  e -= d;
  if (e < sc) {
    a.sig_o[i * sc + e] = (off ? a.osig : a.sig)[s * sc + e];
    return;
  }
  e -= sc;
  if (e < dd) {
    a.A_o[i * dd + e] = (off ? a.oA : a.A)[s * dd + e];
    return;
  }
  e -= dd;
  if (e < dd) {
    a.Ainv_o[i * dd + e] = (off ? a.oAinv : a.Ainv)[s * dd + e];
    return;
  }
  e -= dd;
  if (e < d) {
    a.pc_o[i * d + e] = (off ? a.opc : a.pc)[s * d + e];
    return;
  }
  e -= d;
  if (e < M) {
    a.py_o[i * M + e] = a.cy[ch * M + e];
    return;
  }
  a.rank_o[i] = a.crank[ch];
}

}  // namespace

extern "C" {

int dmo_cmaes_step_record(dmo_ctx* ctx, int kind, void* posterior, uint64_t draw_seed, uint64_t draw_stream, int var_route_mean,
                          int precision, int mean_f32, int cand_f32, const double* parents_x, const double* sigmas, int sigma_cols,
                          const double* A, const double* parents_y, int64_t pop, int d, int M, const double* arz, const int64_t* js,
                          int64_t n_off, int64_t mu, const double* xlb, const double* xub, double* cand_x, double* cand_y,
                          int32_t* cand_rank, double* x_gen, double* y_gen, uint8_t* codes, int64_t* p_idx) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  const char* who = "cmaes_step_record";
  DMO_REQUIRE(parents_x && sigmas && A && parents_y && arz && js && xlb && xub && cand_x && cand_y && cand_rank, "%s: bad arguments", who);
  DMO_REQUIRE(x_gen && y_gen && codes && p_idx, "%s: x_gen, y_gen, codes and p_idx are required", who);
  DMO_REQUIRE(pop >= 2 && n_off >= 1 && mu >= 1 && d >= 1 && d <= 512 && M >= 1 && M <= 16 && (sigma_cols == 1 || sigma_cols == d),
              "%s: bad shape pop=%lld offspring=%lld mu=%lld d=%d M=%d sigma_cols=%d", who, (long long)pop, (long long)n_off, (long long)mu,
              d, M, sigma_cols);
  DMO_REQUIRE(dmo_is_device_ptr(parents_x) && dmo_is_device_ptr(sigmas) && dmo_is_device_ptr(A) && dmo_is_device_ptr(parents_y) &&
                  dmo_is_device_ptr(cand_x) && dmo_is_device_ptr(cand_y) && dmo_is_device_ptr(cand_rank),
              "%s: the parent state (parents_x, sigmas, A, parents_y) and the candidate buffers must be resident on the device", who);
  DMO_REQUIRE(!dmo_is_device_ptr(js), "%s: js is a host array", who);
  const int64_t npick = mu < pop ? mu : pop;  // len(parent_selection)
  for (int64_t i = 0; i < n_off; ++i)
    DMO_REQUIRE(js[i] >= 0 && js[i] < npick, "%s: js[%lld] = %lld is not in [0, %lld)", who, (long long)i, (long long)js[i], (long long)npick);
  DMO_REQUIRE(var_route_mean || kind == DMO_POSTERIOR_GP, "%s: the mean-only predict is the exact GP's (kind %d)", who, kind);
  StepPosterior post;
  DMO_TRY(step_posterior(ctx, who, kind, posterior, draw_seed, draw_stream, var_route_mean != 0, mean_f32 != 0, precision, d, M, &post));
  const int64_t C = n_off, n = n_off + pop;
  In<double> iz, ilb, iub;
  In<int64_t> ijs;
  DMO_TRY(iz.init(ctx, arz, (size_t)C * d));
  DMO_TRY(ijs.init(ctx, js, (size_t)C));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  // 1. the parents' rank, its stable order and the drawn parents (sortMO, CMAES.py:241-262)
  DevBuf<int32_t> prank;
  DevBuf<uint32_t> order;
  DevBuf<int64_t> pidx;
  DMO_TRY(prank.alloc(ctx, pop));
  DMO_TRY(order.alloc(ctx, pop));
  DMO_TRY(pidx.alloc(ctx, C));
  DMO_TRY(rank_nd_device(ctx, parents_y, pop, M, prank.p));
  DMO_TRY(lexsort_device(ctx, prank.p, nullptr, 0, pop, order.p, true));
  DMO_LAUNCH(cmaes_pick_parents_kernel, (unsigned)ceil_div(C, 256), 256, 0, order.p, ijs.d, C, pidx.p);
  // 2. the offspring: sample, global rescale, clip
  DMO_TRY(cmaes_generate_device(ctx, parents_x, sigmas, sigma_cols, A, pidx.p, iz.d, C, d, ilb.d, iub.d, cand_x));
  // 3. their posterior mean (evaluate(x_gen)), then the parents under them (np.vstack((y_gen, parents_y)))
  GpPending gpp;
  DMO_TRY(step_predict(ctx, who, post, cand_x, C, cand_y, nullptr, precision, &gpp));
  bool refined = false;
  DMO_TRY(gp_predict_finish(ctx, post.gp, gpp, &refined));
  if (post.mean_f32) DMO_TRY(prim_round_f32(ctx, cand_y, C * M));
  DMO_CUDA(cudaMemcpyAsync(cand_y + (size_t)C * M, parents_y, (size_t)pop * M * sizeof(double), cudaMemcpyDeviceToDevice, ctx->stream));
  DMO_TRY(copy_out(ctx, x_gen, cand_x, (size_t)C * d * sizeof(double)));
  DMO_TRY(copy_out(ctx, y_gen, cand_y, (size_t)C * M * sizeof(double)));
  // 4. the candidates' rank and the front cut
  DMO_TRY(rank_nd_device(ctx, cand_y, n, M, cand_rank));
  DevBuf<int32_t> cnt, b;
  DevBuf<int64_t> cut;
  DevBuf<uint8_t> code;
  DMO_TRY(cnt.alloc(ctx, n + 1));
  DMO_TRY(b.alloc(ctx, n + 1));
  DMO_TRY(cut.alloc(ctx, 2));
  DMO_TRY(code.alloc(ctx, n));
  DMO_CUDA(cudaMemsetAsync(cnt.p, 0, (size_t)(n + 1) * sizeof(int32_t), ctx->stream));
  DMO_LAUNCH(rank_hist_kernel, (unsigned)ceil_div(n, 256), 256, 0, cand_rank, n, cnt.p);
  DMO_TRY(prim_exclusive_sum_i32(ctx, cnt.p, b.p, n + 1));
  DMO_LAUNCH(front_cut_kernel, (unsigned)std::min<int64_t>(ceil_div(n, 256), 4 * (int64_t)ctx->sm_count), 256, 0, b.p, n, pop, cut.p);
  DMO_LAUNCH(front_codes_kernel, (unsigned)ceil_div(n, 256), 256, 0, cut.p, n, code.p);
  DMO_CHECK_LAUNCH();
  int64_t h_cut[2] = {0, 0};  // the selection's sizes
  DMO_CUDA(cudaMemcpyAsync(h_cut, cut.p, sizeof(h_cut), cudaMemcpyDeviceToHost, ctx->stream));
  DMO_CUDA(dmo_wait(ctx));
  // 5. the mid front's k picks (CMAES.py:200-214)
  const int64_t k = pop - h_cut[0];
  if (k > 0) {
    DevBuf<int64_t> sel;
    if (h_cut[0] > 0) {
      const int64_t nc = h_cut[1] - h_cut[0];
      DevBuf<double> ref, ones;
      DMO_TRY(ref.alloc(ctx, M));
      DMO_TRY(ones.alloc(ctx, (size_t)nc * M));
      DMO_TRY(sel.alloc(ctx, k));
      DMO_LAUNCH(ref_point_kernel, (unsigned)M, kMaxT, 0, cand_y, n, M, cand_f32, ref.p);
      DMO_LAUNCH(fill_kernel, (unsigned)ceil_div(nc * M, 256), 256, 0, ones.p, nc * M, 1.0);
      DMO_TRY(ehvi_select_device(ctx, cand_y, h_cut[0], cand_y + (size_t)h_cut[0] * M, ones.p, nc, M, ref.p, 1, k, sel.p, nullptr));
    }
    DMO_LAUNCH(mid_pick_kernel, (unsigned)ceil_div(k, 256), 256, 0, cut.p, h_cut[0] > 0 ? sel.p : (const int64_t*)nullptr, k, code.p);
    DMO_CHECK_LAUNCH();
  }
  // 6. what the host's update arithmetic needs
  DMO_TRY(copy_out(ctx, codes, code.p, (size_t)n));
  DMO_TRY(copy_out(ctx, p_idx, pidx.p, (size_t)C * sizeof(int64_t)));
  return DMO_OK;
}

int dmo_cmaes_step_apply(dmo_ctx* ctx, const double* parents_x, double* sigmas, int sigma_cols, const double* A, const double* Ainv,
                         const double* pc, int64_t pop, int d, int M, const double* cand_x, const double* cand_y, const int32_t* cand_rank,
                         int64_t n_cand_off, int64_t n_off, const int64_t* off_cand, const int64_t* off_par, const double* off_psucc,
                         const double* off_fac, int64_t n_seg, const int64_t* seg_row, const int64_t* seg_start, const double* ev_fac,
                         const int64_t* next_cand, const int64_t* next_src, const double* xlb, const double* xub, double cc, double ccov,
                         double pthresh, double* parents_x_out, double* sigmas_out, double* A_out, double* Ainv_out, double* pc_out,
                         double* parents_y_out, int32_t* rank_out) {
  if (!ctx) return DMO_ERR_ARG;
  DMO_CUDA(cudaSetDevice(ctx->device));
  const char* who = "cmaes_step_apply";
  const int64_t C = n_cand_off;
  DMO_REQUIRE(parents_x && sigmas && A && Ainv && pc && cand_x && cand_y && cand_rank && next_cand && next_src && xlb && xub &&
                  parents_x_out && sigmas_out && A_out && Ainv_out && pc_out && parents_y_out && rank_out,
              "%s: bad arguments", who);
  DMO_REQUIRE(pop >= 2 && C >= 1 && n_off >= 0 && n_off <= C && n_seg >= 0 && n_seg <= pop && d >= 1 && d <= 512 && M >= 1 &&
                  (sigma_cols == 1 || sigma_cols == d),
              "%s: bad shape", who);
  DMO_REQUIRE(n_off == 0 || (off_cand && off_par && off_psucc && off_fac), "%s: the offspring arrays are required", who);
  DMO_REQUIRE(n_seg == 0 || (seg_row && seg_start && ev_fac), "%s: the event arrays are required", who);
  const void* dev[] = {parents_x, sigmas, A, Ainv, pc, cand_x, cand_y, cand_rank, parents_x_out, sigmas_out, A_out, Ainv_out, pc_out,
                       parents_y_out, rank_out};
  for (const void* p : dev) DMO_REQUIRE(dmo_is_device_ptr(p), "%s: the parent state, the candidates and the outputs must be resident on the device", who);
  const void* host[] = {off_cand, off_par, off_psucc, off_fac, seg_row, seg_start, ev_fac, next_cand, next_src};
  for (const void* p : host) DMO_REQUIRE(!p || !dmo_is_device_ptr(p), "%s: the index and factor arrays are host arrays", who);
  // the outputs are the other half of the double buffer: no gather may read a row already overwritten
  DMO_REQUIRE(parents_x_out != parents_x && sigmas_out != sigmas && A_out != A && Ainv_out != Ainv && pc_out != pc,
              "%s: the outputs must not alias the parent state", who);
  for (int64_t i = 0; i < n_off; ++i)
    DMO_REQUIRE(off_cand[i] >= 0 && off_cand[i] < C && off_par[i] >= 0 && off_par[i] < pop, "%s: offspring %lld out of range", who,
                (long long)i);
  int64_t n_ev = 0;
  if (n_seg > 0) {
    DMO_REQUIRE(seg_start[0] == 0, "%s: seg_start[0] must be 0", who);
    for (int64_t s = 0; s < n_seg; ++s)
      DMO_REQUIRE(seg_row[s] >= 0 && seg_row[s] < pop && seg_start[s + 1] > seg_start[s], "%s: event segment %lld out of range", who,
                  (long long)s);
    n_ev = seg_start[n_seg];
  }
  for (int64_t i = 0; i < pop; ++i) {
    const int64_t ch = next_cand[i], s = next_src[i];
    DMO_REQUIRE(ch >= 0 && ch < C + pop && s >= 0 && s < (ch < C ? n_off : pop), "%s: row %lld of the next parent set out of range", who,
                (long long)i);
  }
  const int sc = sigma_cols;
  In<int64_t> ioc, iop, isr, iss, inc, ins;
  In<double> ips, iof, ief, ilb, iub;
  DMO_TRY(ioc.init(ctx, off_cand, (size_t)n_off));
  DMO_TRY(iop.init(ctx, off_par, (size_t)n_off));
  DMO_TRY(ips.init(ctx, off_psucc, (size_t)n_off));
  DMO_TRY(iof.init(ctx, off_fac, (size_t)n_off));
  DMO_TRY(isr.init(ctx, seg_row, (size_t)n_seg));
  DMO_TRY(iss.init(ctx, seg_start, n_seg ? (size_t)n_seg + 1 : 0));
  DMO_TRY(ief.init(ctx, ev_fac, (size_t)n_ev));
  DMO_TRY(inc.init(ctx, next_cand, (size_t)pop));
  DMO_TRY(ins.init(ctx, next_src, (size_t)pop));
  DMO_TRY(ilb.init(ctx, xlb, d));
  DMO_TRY(iub.init(ctx, xub, d));
  // 1. the chosen offspring's strategy rows, copied from their parents before any update (CMAES.py:330-370)
  DevBuf<double> last, osig, oA, oAinv, opc, z;
  DMO_TRY(last.alloc(ctx, (size_t)n_off * sc));
  DMO_TRY(osig.alloc(ctx, (size_t)n_off * sc));
  DMO_TRY(oA.alloc(ctx, (size_t)n_off * d * d));
  DMO_TRY(oAinv.alloc(ctx, (size_t)n_off * d * d));
  DMO_TRY(opc.alloc(ctx, (size_t)n_off * d));
  DMO_TRY(z.alloc(ctx, (size_t)n_off * d));
  DMO_TRY(gather_rows_device(ctx, sigmas, nullptr, nullptr, iop.d, n_off, sc, last.p));
  DMO_TRY(gather_rows_device(ctx, sigmas, nullptr, nullptr, iop.d, n_off, sc, osig.p));
  DMO_TRY(scale_rows_device(ctx, osig.p, sc, n_off, nullptr, nullptr, iof.d));
  DMO_TRY(gather_rows_device(ctx, A, nullptr, nullptr, iop.d, n_off, (int64_t)d * d, oA.p));
  DMO_TRY(gather_rows_device(ctx, Ainv, nullptr, nullptr, iop.d, n_off, (int64_t)d * d, oAinv.p));
  DMO_TRY(gather_rows_device(ctx, pc, nullptr, nullptr, iop.d, n_off, d, opc.p));
  DMO_TRY(cmaes_step_z_device(ctx, cand_x, ioc.d, parents_x, iop.d, ilb.d, iub.d, last.p, n_off, d, z.p));
  DMO_TRY(cmaes_update_cholesky_device(ctx, oA.p, oAinv.p, opc.p, z.p, ips.d, n_off, d, cc, ccov, pthresh));
  // 2. the parents' success and failure events, in order, on their step sizes (in place: the rows were copied above)
  DMO_TRY(scale_rows_device(ctx, sigmas, sc, n_seg, isr.d, iss.d, ief.d));
  // 3. the next parent set
  Assembly a{parents_x, sigmas, A, Ainv, pc, osig.p, oA.p, oAinv.p, opc.p, cand_x, cand_y, cand_rank, inc.d, ins.d,
             parents_x_out, sigmas_out, A_out, Ainv_out, pc_out, parents_y_out, rank_out};
  const int64_t W = d + sc + 2 * (int64_t)d * d + d + M + 1;
  DMO_LAUNCH(cmaes_assemble_kernel, (unsigned)ceil_div(pop * W, 256), 256, 0, a, pop, C, d, sc, M);
  DMO_CHECK_LAUNCH();
  return DMO_OK;
}

}  // extern "C"
