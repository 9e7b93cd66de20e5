// Small-M ("decode") launchers of the fused packed-int4 linear: the TMA-ring gemvs (M <= 16) and the
// register-streaming warp-MMA kernel (M <= 32).  Everything else goes to the wgmma kernel (api_qbits.cu).
#include "api_qbits.cuh"
#include "gemv_w4.cuh"
#include "gemv_w4s.cuh"
#include "gemv_w4r.cuh"

namespace qb {

struct DecodePlan {
  int P, SPB, span, grid, max_segs;
  int64_t ticket_bytes, partial_bytes;
};

constexpr int64_t kDecodeTicketBytes = 64 * 1024;  // 16384 out-feature blocks (N <= 2M)

static bool decode_applicable(int64_t m, int64_t n, int64_t k) {
  return m >= 1 && m <= 128 && n % 2 == 0 && k % 128 == 0 && (n / 2 + 63) / 64 <= kDecodeTicketBytes / 4;
}

// M <= kGemvMaxM (shapes the ring gemvs do not take): register-streaming warp-MMA kernel (gemv_w4.cuh), several CTAs
// per SM; larger M goes to the wgmma kernel.
constexpr int kGemvMaxM = 8;

static DecodePlan make_decode_plan(int64_t m, int64_t n, int64_t k, int sms) {
  DecodePlan pl;
  pl.P = static_cast<int>((n / 2 + 63) / 64);
  pl.SPB = static_cast<int>(k / 128);  // 128-k stages per out-feature block
  const int total = pl.P * pl.SPB;
  const int ctas_per_sm = m <= 16 ? 3 : 2;
  const int slots = sms * ctas_per_sm;
  int grid = total < slots ? total : slots;
  pl.span = (total + grid - 1) / grid;
  pl.grid = (total + pl.span - 1) / pl.span;
  pl.max_segs = (pl.SPB + pl.span - 1) / pl.span + 1;
  // FIXED-size ticket region: successive launches with different shapes share the workspace, and a ticket must
  // never alias bytes an earlier launch used for partial sums (tickets are the only state that has to stay zero).
  pl.ticket_bytes = kDecodeTicketBytes;
  pl.partial_bytes = static_cast<int64_t>(pl.P) * pl.max_segs * m * 128 * 4;
  return pl;
}

int64_t qbits_small_workspace_bytes(int64_t m, int64_t n, int64_t k) {
  if (!decode_applicable(m, n, k)) return 0;
  // sized for the H100's 132 SMs (the plan is made per device at call time and checked against the size)
  const DecodePlan a = make_decode_plan(m, n, k, kNumSMsH100);
  return a.ticket_bytes + a.partial_bytes;
}

template <typename WT, int MT, bool ZP>
static int launch_gemv(const uint8_t* wq, const void* x, const DecodeParams& p, int grid, cudaStream_t stream) {
  gemv_w4_kernel<WT, MT, ZP><<<grid, kGemvThreads, 0, stream>>>(wq, static_cast<const WT*>(x), p);
  return check_cuda(cudaGetLastError(), "gemv_w4_kernel launch");
}

template <typename WT, bool ZP>
static int launch_gemv_mt(int m, const uint8_t* wq, const void* x, const DecodeParams& p, int grid, cudaStream_t stream) {
  if (m <= 8) return launch_gemv<WT, 1, ZP>(wq, x, p, grid, stream);
  if (m <= 16) return launch_gemv<WT, 2, ZP>(wq, x, p, grid, stream);
  return launch_gemv<WT, 4, ZP>(wq, x, p, grid, stream);
}

// ---------------------------------------------------------------------------------------------
// M <= 8: TMA-ring gemv (gemv_w4s.cuh); whole-K ownership per CTA, no workspace
// ---------------------------------------------------------------------------------------------
constexpr int kGemvSMaxM = 8;
constexpr int kMaxDynSmem = 227 * 1024;

static bool make_gemvs_plan(int64_t m, int64_t n, int64_t k, int group, bool zp, bool coef_aligned, GemvSParams* gp,
                            int* smem_bytes) {
  if (m < 1 || m > kGemvSMaxM || n % 2 != 0 || k % 64 != 0 || group < 16 || (group & (group - 1)) != 0 || k % group != 0)
    return false;
  // the scale / shift runs of a row group are fetched with 16-byte-granular bulk copies starting at any row;
  // shapes where a row of scales is not a multiple of 16 bytes read them with LDG instead (cdepth = 0)
  const int64_t gpr = k / group;
  const bool coef_ring = coef_aligned && (gpr * 2) % 16 == 0 && (!zp || gpr % 16 == 0);
  int kc = 0;
  for (int c = 4096; c >= 1024 && kc == 0; c -= 1024)
    if (k % c == 0) kc = c;
  for (int c = 4096; c >= 64 && kc == 0; c -= 64)
    if (k % c == 0) kc = c;
  if (kc == 0) return false;
  const int nkc = static_cast<int>(k / kc);
  const int stage = 8 * (kc + 64);
  const int64_t coef_arr = 8 * gpr * 2;
  const int64_t x_stride = k * 2 + 16;
  for (int nst = 16; nst >= 3; --nst) {
    // coefficient slots: enough row groups ahead to cover the weight ring
    int cdepth = (nst + nkc - 1) / nkc + 1;
    if (cdepth < 2) cdepth = 2;
    if (!coef_ring) cdepth = 0;
    const int64_t total = 128 + static_cast<int64_t>(nst) * stage + cdepth * 4 * coef_arr + kGemvSRedBytes +
                          (2 * nst + 4 + 2 * cdepth) * 8 + 16 + m * x_stride + 16;
    if (total > kMaxDynSmem) continue;
    gp->KC = kc;
    gp->nkc = nkc;
    gp->nstages = nst;
    gp->stage_bytes = stage;
    gp->x_stride = static_cast<int>(x_stride);
    gp->cdepth = cdepth;
    gp->coef_arr = static_cast<int>(coef_arr);
    *smem_bytes = static_cast<int>(total);
    return true;
  }
  return false;
}

template <typename WT, bool ZP, bool CR, int KO = 0>
static int launch_gemvs_cr(const GemvSParams& p, int grid, int smem_bytes, cudaStream_t stream) {
  int rc = ensure_dyn_smem<gemv_w4s_kernel<WT, ZP, CR, KO>>(kMaxDynSmem);
  if (rc != OK) return rc;
  const bool pdl = test_override(OVR_PDL) != 1;
  return check_cuda(launch_kernel_pdl(gemv_w4s_kernel<WT, ZP, CR, KO>, dim3(grid), dim3(kGemvSThreads), smem_bytes, stream,
                                      pdl, p),
                    "gemv_w4s_kernel launch");
}

template <typename WT, bool ZP, int KO = 0>
static int launch_gemvs(const GemvSParams& p, int grid, int smem_bytes, cudaStream_t stream) {
  if (p.cdepth > 0) return launch_gemvs_cr<WT, ZP, true, KO>(p, grid, smem_bytes, stream);
  if (KO != 0) return fail(ERR_UNSUPPORTED, "knock-outs exist for the coefficient-ring variant only");
  return launch_gemvs_cr<WT, ZP, false, 0>(p, grid, smem_bytes, stream);
}

// ---------------------------------------------------------------------------------------------
// M <= 16, group 64 / 128, K % 1024 == 0: second-generation TMA-ring gemv (gemv_w4r.cuh), compile-time shaped loop
// ---------------------------------------------------------------------------------------------
constexpr int kGemvRMaxM = 16;

struct GemvRPlan {
  int tg, spw, gl, smem_bytes;
  bool lite;  // two CTAs per SM (M <= 2): consecutive launches overlap through programmatic dependent launch
};

static bool make_gemvr_plan(int64_t m, int64_t n, int64_t k, int group, bool zp, bool coef_aligned, int grid, GemvRParams* gp,
                            GemvRPlan* pl) {
  if (m < 1 || m > kGemvRMaxM || n % 16 != 0 || k % 1024 != 0 || (group != 64 && group != 128) || !coef_aligned) return false;
  const int gl = group == 128 ? 1 : 0;
  const int64_t gpr = k / group;
  // coefficient runs of a whole 8-row group travel as bulk copies: 16 * gpr bytes (8 * gpr for zero-points), 16-byte granular
  if (zp && gpr % 2 != 0) return false;
  const int tg = m <= 8 ? 1 : 2;
  const int64_t coef_arr = 8 * gpr * 2;
  const int64_t total_groups = n / 16;
  const int64_t rc = 8 * ((total_groups + grid - 1) / grid);  // rows of the output staging tile per (token, plane)
  const int64_t red = 2 * kGemvRWarps * tg * 128 * 4;
  // The way K is cut (slabs per warp, passes) decides the order of every output's sum, and a column shard must cut it
  // exactly like the full matrix (bit-identical column-parallel results): the choice below depends on M, K and the
  // group size only -- the out-feature dependent buffers are budgeted with a fixed reserve while choosing.
  constexpr int64_t kOutReserve = 24 * 1024;
  constexpr int64_t kMinRing = 48 * 1024;
  pl->lite = false;
  // M <= 2: the "lite" shape -- 2 CTAs per SM (<= 112 KB each): stages of 2048 k, a ring of >= 3 of them.  OPT-IN (test
  // override 7 = 2), not the default: measured on the Llama-3-8B decode step (tools/llama_variants.py, batch 1) the
  // co-resident next kernel's weight stream slows the running one more than the overlap gains: 2.84 ms per step against
  // 1.92 ms for one CTA per SM with programmatic dependent launch (2.24 / 2.31 ms without PDL).
  if (m <= 2 && k % 2048 == 0 && !(gl == 0 && gpr % 2 != 0) && test_override(OVR_GEMV_SHAPE) == 2) {
    constexpr int64_t kLiteSmem = 112 * 1024;
    const int spw = 2, kc = 2048;
    const int nkc = static_cast<int>(k / kc);
    const int64_t stage = 8 * (kc + 64);
    const int64_t x_stride = k * 2 + 16;
    int cdepth = 2;
    const int64_t outs = m * 2 * rc * 2;
    const int64_t base = 128 + red + (2 * 8 + 4 + 2 * cdepth) * 8 + 32 + m * x_stride + 16 + cdepth * 4 * coef_arr + outs;
    int nst = static_cast<int>((kLiteSmem - base) / stage);
    if (nst > 8) nst = 8;
    if (nst >= 3) {
      gp->nxc = 1;
      gp->kx = static_cast<int>(k);
      gp->nkc = nkc;
      gp->nstages = nst;
      gp->cdepth = cdepth;
      gp->coef_arr = static_cast<int>(coef_arr);
      gp->x_stride = static_cast<int>(x_stride);
      gp->rc = static_cast<int>(rc);
      pl->tg = 1;
      pl->spw = spw;
      pl->gl = gl;
      pl->lite = true;
      pl->smem_bytes = static_cast<int>(base + nst * stage);
      return true;
    }
  }
  for (int spw = 4; spw >= (1 << gl); spw >>= 1) {
    if (k % (spw * 1024) != 0) continue;
    if ((spw >> gl) == 2 && gpr % 2 != 0) continue;  // the pair of groups is read with one 32-bit load
    const int kc = spw * 1024;
    const int nk = static_cast<int>(k / kc);
    const int64_t stage = 8 * (kc + 64);
    for (int nxc = 1; nxc <= nk; ++nxc) {
      if (nk % nxc != 0) continue;
      // several passes cost a pipeline drain each: worth it for M <= 8 only, where this kernel is the only one whose
      // k-order does not depend on the shard
      if (nxc > 1 && m > 8) break;
      const int nkc = nk / nxc;
      const int64_t kx = k / nxc;
      const int64_t x_stride = kx * 2 + 16;
      const int64_t x_bytes = m * x_stride;
      for (int nst = 16; nst >= 2; --nst) {
        // choosing: out-feature dependent buffers (output staging, partial sums of the passes, resident coefficient slots
        // of a multi-pass kernel) are budgeted with fixed reserves, so that the cut of K never depends on N
        int cdepth = (nst + nkc - 1) / nkc + 1;
        if (cdepth < 2) cdepth = 2;
        const int64_t coef_sel = nxc > 1 ? 16 * 1024 : cdepth * 4 * coef_arr;
        const int64_t base = 128 + red + (2 * nst + 4 + 2 * 64) * 8 + 32 + x_bytes + 16;
        if (base + coef_sel + nst * stage + kOutReserve > kMaxDynSmem) continue;
        // too shallow a ring: more passes (smaller x) or narrower stages -- where that choice exists (M <= 8)
        if (nst * stage < kMinRing && m <= 8) break;
        // the actual out-feature dependent part may only cost ring depth
        if (nxc > 1) cdepth = static_cast<int>(rc / 8);  // every row group of the CTA keeps its coefficient slot
        if (cdepth > 64) return false;
        const int64_t outs = m * 2 * rc * 2 + (nxc > 1 ? (rc / 8) * tg * 128 * 4 : 0);
        const int64_t fixed = base + cdepth * 4 * coef_arr + outs;
        int nst_fit = nst;
        while (nst_fit >= 2 && fixed + nst_fit * stage > kMaxDynSmem) --nst_fit;
        if (nst_fit < 2) return false;
        gp->nxc = nxc;
        gp->kx = static_cast<int>(kx);
        gp->nkc = nkc;
        gp->nstages = nst_fit;
        gp->cdepth = cdepth;
        gp->coef_arr = static_cast<int>(coef_arr);
        gp->x_stride = static_cast<int>(x_stride);
        gp->rc = static_cast<int>(rc);
        pl->tg = tg;
        pl->spw = spw;
        pl->gl = gl;
        pl->smem_bytes = static_cast<int>(fixed + nst_fit * stage);
        return true;
      }
    }
  }
  return false;
}

template <typename WT, bool ZP, int TG, int SPW, int GL, bool MPASS, int NP>
static int launch_gemvr_inst(const GemvRParams& p, int grid, int smem_bytes, cudaStream_t stream) {
  int rc = ensure_dyn_smem<gemv_w4r_kernel<WT, ZP, TG, SPW, GL, MPASS, NP>>(kMaxDynSmem);
  if (rc != OK) return rc;
  const bool pdl = test_override(OVR_PDL) != 1;
  return check_cuda(launch_kernel_pdl(gemv_w4r_kernel<WT, ZP, TG, SPW, GL, MPASS, NP>, dim3(grid), dim3(gemvr_threads(NP)),
                                      smem_bytes, stream, pdl, p),
                    "gemv_w4r_kernel launch");
}

template <typename WT, bool ZP, int TG, bool MPASS>
static int launch_gemvr_shape(const GemvRParams& p, const GemvRPlan& pl, int grid, cudaStream_t stream) {
  if (pl.gl == 1) {
    if (pl.spw == 4) return launch_gemvr_inst<WT, ZP, TG, 4, 1, MPASS, 8>(p, grid, pl.smem_bytes, stream);
    return launch_gemvr_inst<WT, ZP, TG, 2, 1, MPASS, 8>(p, grid, pl.smem_bytes, stream);
  }
  if (pl.spw == 4) return launch_gemvr_inst<WT, ZP, TG, 4, 0, MPASS, 8>(p, grid, pl.smem_bytes, stream);
  if (pl.spw == 2) return launch_gemvr_inst<WT, ZP, TG, 2, 0, MPASS, 8>(p, grid, pl.smem_bytes, stream);
  return launch_gemvr_inst<WT, ZP, TG, 1, 0, MPASS, 8>(p, grid, pl.smem_bytes, stream);
}

template <typename WT, bool ZP>
static int launch_gemvr(const GemvRParams& p, const GemvRPlan& pl, int grid, cudaStream_t stream) {
  if (pl.lite) {
    if (pl.gl == 1) return launch_gemvr_inst<WT, ZP, 1, 2, 1, false, 4>(p, grid, pl.smem_bytes, stream);
    return launch_gemvr_inst<WT, ZP, 1, 2, 0, false, 4>(p, grid, pl.smem_bytes, stream);
  }
  if (pl.tg == 1) {
    if (p.nxc > 1) return launch_gemvr_shape<WT, ZP, 1, true>(p, pl, grid, stream);
    return launch_gemvr_shape<WT, ZP, 1, false>(p, pl, grid, stream);
  }
  return launch_gemvr_shape<WT, ZP, 2, false>(p, pl, grid, stream);
}

// Host-only: how the ring gemv would cut K for this problem on a grid of `grid` CTAs (0 = it does not take the problem).
// out[0..4] = slabs per warp, passes over K, ring stages, token groups, dynamic shared memory bytes.
int qbits_ring_plan(int64_t m, int64_t n, int64_t k, int group, int zp, int grid, int* out) {
  GemvRParams gp{};
  GemvRPlan pl{};
  const int64_t groups = n / 16;
  const int g = static_cast<int>(groups < grid ? (groups > 0 ? groups : 1) : grid);
  if (!make_gemvr_plan(m, n, k, group, zp != 0, true, g, &gp, &pl)) return 0;
  out[0] = pl.spw;
  out[1] = gp.nxc;
  out[2] = gp.nstages;
  out[3] = pl.tg;
  out[4] = pl.smem_bytes;
  return 1;
}

// Returns OK and sets *handled when one of the small-M kernels took the problem; *handled = false (and OK) when the
// caller should use the general kernel; a non-zero status is a launch / argument failure.
int qbits_small_dispatch(const QbitsArgs& q, bool* handled) {
  *handled = false;
  const int64_t m = q.m, n = q.n, k = q.k;
  const int route = test_override(OVR_INT4_ROUTE);
  if (route == ROUTE_INT4_GENERAL) return OK;
  cudaStream_t st = q.stream;
  const bool zp = q.shift_is_int != 0;
  const int dbg = debug_flags();

  if (route == ROUTE_AUTO || route == ROUTE_INT4_RING2) {
    GemvRParams rp{};
    GemvRPlan rpl{};
    const bool coef_aligned = aligned16(q.scale) && aligned16(q.shift);
    const int64_t r_groups = n / 16;
    const int r_grid = static_cast<int>(r_groups < current_sm_count() ? (r_groups > 0 ? r_groups : 1) : current_sm_count());
    bool out_aligned = aligned16(q.out) && q.ld % 8 == 0 && q.col0 % 8 == 0;
    for (int pq = 1; pq < q.g.n_out; ++pq) out_aligned = out_aligned && aligned16(q.g.out_peer[pq]);
    if (out_aligned && aligned16(q.a) &&
        make_gemvr_plan(m, n, k, q.group, zp, coef_aligned, r_grid, &rp, &rpl)) {
      rp.wq = q.packed;
      rp.scale = q.scale;
      rp.shift = q.shift;
      rp.bias = q.bias;
      rp.x = q.a;
      rp.out = q.out;
      rp.g = q.g;
      rp.ld = static_cast<int>(q.ld);
      rp.col0 = static_cast<int>(q.col0);
      rp.M = static_cast<int>(m);
      rp.N = static_cast<int>(n);
      rp.K = static_cast<int>(k);
      rp.trace = debug_trace();
      const int grid = r_grid;
      set_kernel_family(3);
      *handled = true;
      return dispatch_act16_zp(q.dtype, q.shift_is_int, [&](auto act, auto ZP) {
        return launch_gemvr<typename decltype(act)::WT, ZP>(rp, rpl, grid, st);
      });
    }
    if (route == ROUTE_INT4_RING2) return fail(ERR_UNSUPPORTED, "qbits_mm: the second-generation ring gemv does not take this problem");
  }

  if (route == ROUTE_AUTO || route == ROUTE_INT4_RING) {
    GemvSParams gp{};
    int smem_bytes = 0;
    const bool coef_aligned = aligned16(q.scale) && aligned16(q.shift);
    if (aligned16(q.a) && make_gemvs_plan(m, n, k, q.group, zp, coef_aligned, &gp, &smem_bytes)) {
      gp.wq = q.packed;
      gp.scale = q.scale;
      gp.shift = q.shift;
      gp.bias = q.bias;
      gp.x = q.a;
      gp.out = q.out;
      gp.g = q.g;
      gp.ld = static_cast<int>(q.ld);
      gp.col0 = static_cast<int>(q.col0);
      gp.M = static_cast<int>(m);
      gp.N = static_cast<int>(n);
      gp.K = static_cast<int>(k);
      gp.group = q.group;
      gp.group_log2 = q.group_log2;
      gp.dbg = dbg;
      gp.trace = debug_trace();
      const int pm = test_override(OVR_GEMV_PRODUCER);
      gp.pmode = pm == 0 ? kGemvSDefaultProducer : pm - 1;
      const int64_t half_n = n / 2;
      const int grid = static_cast<int>(half_n < current_sm_count() ? half_n : current_sm_count());
      set_kernel_family(3);
      *handled = true;
#ifdef QB_DEVELOPER_KNOCKOUTS
      // the knock-out variants exist for bf16 with a float shift only
      if (q.dtype == DT_BF16 && !zp) {
        if ((dbg & 3) == 1) return launch_gemvs<__nv_bfloat16, false, 1>(gp, grid, smem_bytes, st);
        if ((dbg & 3) == 2) return launch_gemvs<__nv_bfloat16, false, 2>(gp, grid, smem_bytes, st);
        if ((dbg & 3) == 3) return launch_gemvs<__nv_bfloat16, false, 3>(gp, grid, smem_bytes, st);
      }
#endif
      return dispatch_act16_zp(q.dtype, q.shift_is_int, [&](auto act, auto ZP) {
        return launch_gemvs<typename decltype(act)::WT, ZP>(gp, grid, smem_bytes, st);
      });
    }
    if (route == ROUTE_INT4_RING) return fail(ERR_UNSUPPORTED, "qbits_mm: the ring gemv does not take this problem");
  }

  // register-streaming gemv: M <= 8 (M <= 32 on request), one plain [M, N] output (no fused gather)
  const bool want_gemv = route == ROUTE_INT4_GEMV || (route == ROUTE_AUTO && m <= kGemvMaxM);
  if (!want_gemv) return OK;
  if (route == ROUTE_INT4_GEMV && m > 32) return fail(ERR_UNSUPPORTED, "qbits_mm: the warp-MMA gemv takes M <= 32");
  const bool gemv_ok = decode_applicable(m, n, k) && q.workspace != nullptr && q.g.n_out == 1 && q.ld == q.n &&
                       q.col0 == 0 && q.group % 16 == 0 && reinterpret_cast<uintptr_t>(q.a) % 8 == 0;
  DecodePlan pl = make_decode_plan(m, n, k, current_sm_count());
  if (!gemv_ok || pl.ticket_bytes + pl.partial_bytes > q.workspace_bytes || reinterpret_cast<uintptr_t>(q.workspace) % 256 != 0) {
    if (route != ROUTE_AUTO) return fail(ERR_UNSUPPORTED, "qbits_mm: the warp-MMA gemv needs K %% 128 == 0, a plain output and a large enough workspace");
    return OK;
  }
  DecodeParams d{};
  d.scale = q.scale;
  d.shift = q.shift;
  d.bias = q.bias;
  d.out = q.out;
  d.g = q.g;
  d.ld = static_cast<int>(q.ld);
  d.col0 = static_cast<int>(q.col0);
  d.tickets = static_cast<int*>(q.workspace);
  d.partials = reinterpret_cast<float*>(static_cast<uint8_t*>(q.workspace) + pl.ticket_bytes);
  d.M = static_cast<int>(m);
  d.N = static_cast<int>(n);
  d.K = static_cast<int>(k);
  d.group = q.group;
  d.group_log2 = q.group_log2;
  d.shift_is_int = q.shift_is_int;
  d.P = pl.P;
  d.SPB = pl.SPB;
  d.span = pl.span;
  d.max_segs = pl.max_segs;
  d.dbg = dbg;
  *handled = true;
  set_kernel_family(3);
  return dispatch_act16_zp(q.dtype, q.shift_is_int, [&](auto act, auto ZP) {
    return launch_gemv_mt<typename decltype(act)::WT, ZP>(static_cast<int>(m), q.packed, q.a, d, pl.grid, st);
  });
}

}  // namespace qb
