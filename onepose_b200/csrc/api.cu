// C ABI of the H100-native GATsSPG matcher (see include/onepose_b200.h).
// Host-side state: packed weights, per-object constants, chunk workspace, launch sequence.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/onepose_b200.h"
#include "common.cuh"
#include "gemm_common.cuh"
#include "gemm_tc.cuh"
#include "host_util.cuh"
#include "kernels_aux.cuh"
#include "kv_state_tc.cuh"

namespace opb {

constexpr int kDefaultChunk = 32;   // frames pushed through the GNN together (measured: 4 -> 1340, 8 -> 1650, 16 -> 2390, 32 -> 2550 frames/s)
constexpr int kQPassFrames = 16;    // granularity of the query-side layer-1 pass when the queries stream in from the host
constexpr double kMinScaleFactor = 2.0 * 1.4426950408889634 / 126.0;   // ~0.0229: smallest scale_factor opb_create accepts

static bool g_pdl = true;
static int g_ws_fill = -1;     // >= 0: byte value written into every fresh allocation that the algorithm does not require to be zero
int ws_fill_byte() { return g_ws_fill; }
bool pdl_enabled() { return g_pdl; }
void set_pdl_enabled(bool on) { g_pdl = on; }

struct AttnLayerW {       // one AttentionPropagation (reference GATs_SuperGlue.py:104-113)
  PlaneBuf wqkv;          // [768,256]  rows: Q | K | V, head-contiguous output channels
  DevBuf bqkv;            // [768]
  PlaneBuf w0a;           // [512,256]  mlp.0.weight[:, :256]
  PlaneBuf w0m;           // [512,256]  mlp.0.weight[:, 256:] @ merge.weight (head-contiguous inputs): A operand of the G-fold GEMM
  DevBuf b0f;             // [512] = mlp.0.weight[:,256:] @ merge.bias + mlp.0.bias
  PlaneBuf w1;            // [256,512]  mlp.3.weight
  DevBuf b1;              // [256]
};

struct ObjectState {      // per-object constants: the handle's current object (opb_set_object) or one opb_add_object registration
  int M = 0, Lf = 0, m_pad = 0;
  DevBuf leaves;          // fp32 [M*Lf, 256] point-major
  PlaneBuf db;            // [m_pad, 256]
  DevBuf s2;              // [4][M*Lf]: leaf logits, valid while s2_ready (they depend on the weights)
  PlaneBuf xo;            // [m_pad, 256]: 3D-point state entering layer 2 (object prologue), valid while prologue_ready
  bool s2_ready = false;
  bool prologue_ready = false;
};

constexpr int kCurrentObject = -1;   // key of opb_set_object's object in opb_matcher::objects; opb_add_object's ids count up from 0

}  // namespace opb

using namespace opb;

struct opb_matcher : Handle {
  opb_config cfg{};
  bool weights_ready = false;
  int num_sms = 132;      // multiprocessors of the device (opb_create reads it; 132 on an H100 SXM)
  // packed weights
  AttnLayerW attn[8];
  DevBuf wa2, wa3;        // [4][256] each (GATs: W a[:256], W a[256:])
  PlaneBuf wlin;          // [4][256][256]: W^T of the GATs layers (with_linear_transform only)
  PlaneBuf wf;            // final_proj [256,256]
  DevBuf bf;
  PlaneBuf eye;           // [256,256] identity, fp16-split (residual as an identity K-block of the mlp.3 GEMM)
  std::map<int, ObjectState> objects;           // opb_add_object registrations by id; opb_set_object's object under kCurrentObject
  int next_object_id = 0;
  // workspace (chunk)
  int chunk_frames = 0;   // user override
  int ws_frames = 0, ws_N = 0, ws_m_pad = 0;
  DevBuf tab;             // ChunkTable of the chunk in flight (written by assemble_layout)
  bool hoist = true;      // evaluate the frame-invariant layers once per object (object_prologue)
  int kv_two_pass = 1;    // k,v projection as A_hi.(B_hi + B_lo): its output is one fp16 plane, the A_lo term is below that rounding
  PlaneBuf x, qp, pn, g, xq, bd, lin_a, lin_b;
  DevBuf kvt;             // fp16 [rows, 512]
  DevBuf hid, kvpart, kmean, statpart, mu, rstd, rowsum_part, colsum_part, rowsum, colsum, rowbest, colbest;
  DevBuf range_flag;
  int* range_host = nullptr;                    // pinned copy of the flag, written at the end of every opb_forward
  bool range_pending = false;
  // host-call staging
  DevBuf st_q, st_m0, st_m1, st_s0, st_s1, st_conf, st_len;
  cudaStream_t copy_stream = nullptr;          // opb_forward_host: H2D of chunk i+1 overlaps the compute of chunk i
  std::vector<cudaEvent_t> h2d_ev;              // one per piece; consumed by the chunk loop of opb_forward
  int h2d_pending = 0;
  int last_launches = 0;                        // launches of the last completed forward
  // test hook (opb_debug_set_stop / opb_debug_read): the next forward stops after step dbg_step of GNN layer dbg_layer
  int dbg_layer = -1, dbg_step = 0;
  int dbg_chunk = 0, dbg_piece = 0;             // ... in chunk dbg_chunk (and sub-batch dbg_piece of the hoisted query pass)
  int pass_chunk = 0, pass_piece = -1;          // the pass being enqueued: its chunk, its query-pass sub-batch (-1: none)
  bool dbg_stopped = false;                     // the last forward stopped there; dbg_L / dbg_x are the layout and X of that pass
  Layout dbg_L{};
  XView dbg_x{};
  ~opb_matcher() {
    for (auto e : h2d_ev) cudaEventDestroy(e);
    if (copy_stream) cudaStreamDestroy(copy_stream);
    if (range_host) cudaFreeHost(range_host);
  }
};

namespace opb {

// One GATsSPG GEMM; its profile name tells the epilogue and the shape (bench.py selects on "gemm epi1 ", ...).
static int gemm(opb_matcher* m, const GemmProblem& p, cudaStream_t st, double flops, const char* what) {
  char tag[96] = "";
  if (m->timeline.on) snprintf(tag, sizeof tag, "gemm epi%d n%d k%d %s", p.epi, p.n_out, p.K1 + p.K2, what);
  return run_gemm(m, p, st, flops, what, tag);
}

// Sized for chunks of `frames` frames, N query points and 3D segments of m_pad rows (the largest object of a call); only grows.
static int ensure_workspace(opb_matcher* m, int frames, int N, int m_pad) {
  if (frames <= m->ws_frames && N <= m->ws_N && m_pad <= m->ws_m_pad) return 0;
  frames = std::max(frames, m->ws_frames);
  N = std::max(N, m->ws_N);
  m_pad = std::max(m_pad, m->ws_m_pad);
  const int n_pad = round_up(N, kSegPad);
  const size_t R = (size_t)n_pad + m_pad;
  const size_t rows = R * frames;
  const size_t S = 2 * (size_t)frames;
  CK(m, m->x.ensure(rows * kD));
  CK(m, m->qp.ensure(rows * kD));
  CK(m, m->pn.ensure(rows * kD));
  CK(m, m->g.ensure(S * 512 * kD));
  CK(m, m->bd.ensure(S * kD * kD, true));          // block-diagonal state operand: off-diagonal blocks stay zero for the buffer's lifetime
  CK(m, m->xq.ensure((size_t)frames * n_pad * kD));
  CK(m, m->kvt.ensure(rows * 512 * sizeof(__half)));
  CK(m, m->hid.ensure(rows * 512 * sizeof(float)));
  CK(m, m->kvpart.ensure(rows / 256 * kHeads * kKVPartial * sizeof(float)));
  CK(m, m->kmean.ensure(S * kD * sizeof(float)));
  CK(m, m->statpart.ensure(rows / 32 * 512 * 2 * sizeof(float)));
  CK(m, m->mu.ensure(S * 512 * sizeof(float)));
  CK(m, m->rstd.ensure(S * 512 * sizeof(float)));
  CK(m, m->rowsum.ensure((size_t)frames * n_pad * sizeof(float)));
  CK(m, m->rowsum_part.ensure((size_t)frames * (m_pad / 256) * 2 * n_pad * sizeof(float)));
  CK(m, m->colsum_part.ensure((size_t)frames * (n_pad / 32) * m_pad * sizeof(float)));
  CK(m, m->colsum.ensure((size_t)frames * m_pad * sizeof(float)));
  CK(m, m->rowbest.ensure((size_t)frames * n_pad * sizeof(unsigned long long)));
  CK(m, m->colbest.ensure((size_t)frames * m_pad * sizeof(unsigned long long)));
  CK(m, m->range_flag.ensure(sizeof(int), true));
  CK(m, m->tab.ensure(sizeof(ChunkTable)));
  if (m->cfg.with_linear_transform) {
    CK(m, m->lin_a.ensure((size_t)frames * m_pad * kD));
    CK(m, m->lin_b.ensure((size_t)frames * m_pad * kD));
  }
  // (re)allocation fills ran on the legacy stream: order them against the caller's (possibly non-blocking) stream once
  CK(m, cudaDeviceSynchronize());
  m->ws_frames = frames;
  m->ws_N = N;
  m->ws_m_pad = m_pad;
  return 0;
}

static ChunkTable* tab_dev(const opb_matcher* m) { return m->tab.as<ChunkTable>(); }

// Test hook: layer ids of opb_debug_set_stop.  0..11 are the GNN layers of a chunk, kTailLayer the tail; with hoisting, layer 1
// is the compact query-side pass and the object prologue's layers 0 and 1 are kPrologueLayer + 0 / + 1.
constexpr int kTailLayer = 12;
constexpr int kPrologueLayer = 16;
constexpr int kStopped = 1;      // internal return code of a forward that reached the stop (never returned by the C ABI)

// True when the forward is to stop after step `step` of `layer` (of chunk dbg_chunk, and of sub-batch dbg_piece in the hoisted
// query pass; the object prologue belongs to no chunk); then records the pass for opb_debug_read.  A host-side comparison only:
// the launch sequence is the same with the hook off.
static bool stop_here(opb_matcher* m, int layer, int step, const Layout& L, XView x) {
  if (layer != m->dbg_layer || step != m->dbg_step) return false;
  if (layer < kPrologueLayer && (m->pass_chunk != m->dbg_chunk || (m->pass_piece >= 0 && m->pass_piece != m->dbg_piece))) return false;
  m->dbg_stopped = true;
  m->dbg_L = L;
  m->dbg_x = x;
  return true;
}

// Frame b of a chunk matches against its object's rows `o`.
static void table_frame(ChunkTable& t, int b, const ObjectState& o, bool hoist) {
  t.obj[b] = FrameObject{hoist ? o.xo.hi.as<__half>() : o.db.hi.as<__half>(), hoist ? o.xo.lo.as<__half>() : o.db.lo.as<__half>(),
                         o.leaves.as<float>(), o.s2.as<float>()};
  t.mlen[b] = o.M;
}

// GATs groups of a chunk: runs of consecutive frames of one object, cut at kGatsFramesPerWarp frames.  With one object these
// are [0, 16), [16, 32), ...; frames of an object placed next to each other in a call share their leaf reads.
static void make_groups(GatsGroups& g, const ObjectState* const* fobj, int fb) {
  g.n = 0;
  for (int b = 0; b < fb; ++b) {
    if (b == 0 || fobj[b] != fobj[b - 1] || b - g.g[g.n - 1].b_begin == kGatsFramesPerWarp)
      g.g[g.n++] = GatsGroup{fobj[b]->leaves.as<float>(), fobj[b]->s2.as<float>(), b, b, fobj[b]->M, 0};
    g.g[g.n - 1].b_end = b + 1;
  }
}

// One GATs layer on the 3D-point segments of `x` (layout L); frame b aggregates the leaves of its object (chunk table, already
// on the device; `groups` for the 8-leaf kernel), `Lf` leaves per point.
static int run_gats(opb_matcher* m, const Layout& L, XView x, int layer, int Lf, const GatsGroups& groups, cudaStream_t st) {
  const int gi = (layer % kPrologueLayer) / 3;
  const long long warps = (long long)L.M * L.B;
  if (warps == 0) return 0;
  const bool lin = m->cfg.with_linear_transform != 0;
  GatsOut out{lin ? m->lin_a.hi.as<__half>() : x.hi, lin ? m->lin_a.lo.as<__half>() : x.lo, lin ? 1 : 0};
  const float* wa3 = m->wa3.as<float>() + gi * kD;
  const ChunkTable* tab = tab_dev(m);
  if (Lf == 8) {   // leaves loaded once per point and reused across the frames of a group (frame-independent results)
    const long long w8 = (long long)L.M * groups.n;
    LAUNCH(m, st, "gats_aggregate", gats_aggregate_frames8, dim3((unsigned)((w8 * 32 + 255) / 256)), dim3(256), 0, st, (const __half*)x.hi,
           (const __half*)x.lo, L, groups, gi, wa3, (int)m->cfg.include_self, (int)m->cfg.additional, 0.2f, out);
  } else {
    LAUNCH(m, st, "gats_aggregate", gats_aggregate, dim3((unsigned)((warps * 32 + 255) / 256)), dim3(256), 0, st, (const __half*)x.hi,
           (const __half*)x.lo, L, tab, Lf, gi, wa3, (int)m->cfg.include_self, (int)m->cfg.additional, 0.2f, out);
  }
  if (stop_here(m, layer, 0, L, x)) return kStopped;
  if (!lin) return 0;
  // with_linear_transform (GATs.py:56-57,64-65): t = pre . W on the tensor cores over the compact 3D rows, then ELU (+ h3)
  Layout Lc{};
  Lc.B = L.B; Lc.N = 0; Lc.M = L.M; Lc.n_pad = 0; Lc.m_pad = L.m_pad; Lc.R = L.m_pad; Lc.mlen = L.mlen;
  GemmProblem p{};
  p.L = Lc; p.batch = 1; p.rows = Lc.rows();
  p.a1 = m->lin_a.c(kD); p.K1 = kD; p.b1 = m->wlin.c(kD, (size_t)gi * kD * kD); p.n_out = kD;
  p.epi = EPI_BIAS_PLANES; p.out = m->lin_b.m(kD);
  if (int rc = gemm(m, p, st, 2.0 * L.B * (double)L.M * kD * kD, "gats.W")) return rc;
  const long long n = (long long)L.B * L.M * 32;
  LAUNCH(m, st, "gats_lin_finish", gats_lin_finish, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, st, (const __half*)m->lin_b.hi.as<__half>(),
         (const __half*)m->lin_b.lo.as<__half>(), x.hi, x.lo, L, (int)(m->cfg.include_self && m->cfg.additional));
  if (stop_here(m, layer, 1, L, x)) return kStopped;
  return 0;
}

// One AttentionPropagation layer (reference GATs_SuperGlue.py:55-64, :104-113) on every segment of `x`:
// both sides of all frames in ONE set of 8 launches (the layer's weights are shared by the two sides).
static int run_attn_layer(opb_matcher* m, const Layout& L, XView x, int layer, AttnLayerW& W, int cross, cudaStream_t st) {
  const int rows = L.rows();
  const int S = L.segs();
  const double valid_rows = (double)L.B * (L.N + L.M);
  // (1) k,v projection (:96-99), rows [256, 768) of the packed weight; epilogue: elu+1 on K, pad rows zeroed, ONE fp16 plane
  //     kvt[rows, 512] = fp16(64 * [elu1(K) | V]) -- the single-pass operands of the state kernel
  GemmProblem pk{};
  pk.L = L; pk.batch = 1; pk.rows = rows;
  pk.a1 = x.c(kD); pk.K1 = kD; pk.b1 = W.wqkv.c(kD, (size_t)256 * kD); pk.n_out = 512;
  pk.bias = W.bqkv.as<float>() + 256;
  pk.epi = EPI_QKV; pk.out = Planes{m->kvt.as<__half>(), m->kvt.as<__half>(), 512};
  pk.a_hi_only = m->kv_two_pass;
  if (int rc = gemm(m, pk, st, 2.0 * valid_rows * 512 * kD, "kv_proj")) return rc;
  if (stop_here(m, layer, 0, L, x)) return kStopped;
  // (2) linear-attention state of every segment (:71-78): per-row-group partial states on the tensor cores ...
  const KvGroups G = kv_groups_for(L, m->num_sms);
  if (int rc = launched(m, st, "kv_state_h", launch_kv_state_h(m->kvt.as<__half>(), L, G, m->kvpart.as<float>(), st))) return rc;
  if (stop_here(m, layer, 1, L, x)) return kStopped;
  // ... reduced per segment into Kmean and the block-diagonal operand of the G fold (indexed by DESTINATION segment)
  LAUNCH(m, st, "kv_state_reduce", kv_state_reduce, dim3(S * kHeads, (kKVPartial + 255) / 256), dim3(256), 0, st, (const float*)m->kvpart.as<float>(), L,
         G, cross, m->kmean.as<float>(), m->bd.hi.as<__half>(), m->bd.lo.as<__half>());
  if (stop_here(m, layer, 2, L, x)) return kStopped;
  // (3) q projection; epilogue: elu+1 and the per-head normaliser with the SOURCE segment's K mean -> Q' planes (:78-79)
  GemmProblem pq{};
  pq.L = L; pq.batch = 1; pq.rows = rows;
  pq.a1 = x.c(kD); pq.K1 = kD; pq.b1 = W.wqkv.c(kD); pq.n_out = 256; pq.bias = W.bqkv.as<float>();
  pq.epi = EPI_QSCALE; pq.kmean = m->kmean.as<float>(); pq.cross = cross; pq.out = m->qp.m(kD);
  if (int rc = gemm(m, pq, st, 2.0 * valid_rows * 256 * kD, "q_proj")) return rc;
  if (stop_here(m, layer, 3, L, x)) return kStopped;
  // (4) dynamic weight G[s] = W0m . blockdiag(KVmean_src(s))^T  -- merge and the message half of mlp.0 folded into one
  //     per-segment [512, 256] weight (4 x 64x64x512 MACs per segment), as a batched wgmma GEMM over the segments
  GemmProblem pg{};
  pg.batch = S; pg.rows = 512; pg.n_out = kD; pg.K1 = kD;
  pg.a1 = W.w0m.c(kD); pg.a_batch_rows = 0;
  pg.b1 = m->bd.c(kD); pg.b_batch_rows = kD;
  pg.epi = EPI_BIAS_PLANES; pg.out = m->g.m(kD);
  if (int rc = gemm(m, pg, st, 2.0 * S * 512.0 * kD * kDh, "g_fold")) return rc;
  if (stop_here(m, layer, 4, L, x)) return kStopped;
  // (5) hidden = mlp.0([x ; message]) = [x | Q'] . [W0a | G_seg]^T + b   (:101,:113,:122); epilogue also emits the InstanceNorm
  //     partial sums (:126)
  GemmProblem p2{};
  p2.L = L; p2.batch = 1; p2.rows = rows;
  p2.a1 = x.c(kD); p2.K1 = kD; p2.b1 = W.w0a.c(kD);
  p2.a2 = m->qp.c(kD); p2.K2 = kD; p2.b2 = m->g.c(kD); p2.b2_per_seg = 1;
  p2.n_out = 512; p2.bias = W.b0f.as<float>(); p2.c = m->hid.as<float>(); p2.ldc = 512;
  p2.epi = EPI_F32_STATS; p2.statpart = m->statpart.as<float>();
  if (int rc = gemm(m, p2, st, 2.0 * valid_rows * 512 * 512, "mlp0")) return rc;
  if (stop_here(m, layer, 5, L, x)) return kStopped;
  // (6) InstanceNorm statistics per segment (:126)
  LAUNCH(m, st, "in_stats_final", in_stats_final, dim3(S, 16), dim3(32, kStatSlices), 0, st, (const float*)m->statpart.as<float>(), L, m->mu.as<float>(),
         m->rstd.as<float>());
  if (stop_here(m, layer, 6, L, x)) return kStopped;
  // (7) x <- x + mlp.3(ReLU(IN(hidden)))  (:122, :59/:64): the converters form hn inside the GEMM, the residual is an identity K-block
  GemmProblem p3{};
  p3.L = L; p3.batch = 1; p3.rows = rows;
  p3.K1 = 512; p3.b1 = W.w1.c(512); p3.n_out = 256; p3.bias = W.b1.as<float>();
  p3.epi = EPI_BIAS_PLANES; p3.out = x.m(kD);
  p3.a2 = x.c(kD); p3.K2 = kD; p3.b2 = m->eye.c(kD); p3.b2_lo_zero = 1;
  p3.a_conv = 1; p3.a_raw = m->hid.as<float>(); p3.a_raw_ld = 512; p3.mu = m->mu.as<float>(); p3.rstd = m->rstd.as<float>();
  if (int rc = gemm(m, p3, st, 2.0 * valid_rows * 256 * 512, "mlp3")) return rc;
  return stop_here(m, layer, 7, L, x) ? kStopped : 0;
}

// Object prologue: GNN layers 0 (GATs) and the 3D side of layer 1 (self-attention) depend only on the per-object
// constants (reference GATs_SuperGlue.py:50-54 and :60-64 with src1 = desc3d_db), not on the query frame.  They are
// evaluated ONCE PER OBJECT -- on a single copy of the object's rows, by the first call that uses the object after
// opb_set_object / opb_add_object / opb_finalize_weights (it needs the chunk workspace) -- and shared by every frame of every
// later call, like the leaf logits s2.  Result: o.xo = 3D-point state entering layer 2.
static int object_prologue(opb_matcher* m, ObjectState& o, cudaStream_t st) {
  Layout Lo{};
  Lo.B = 1; Lo.N = 0; Lo.M = o.M; Lo.n_pad = 0; Lo.m_pad = o.m_pad; Lo.R = o.m_pad;
  ChunkTable t{};
  table_frame(t, 0, o, /*hoist=*/false);
  GatsGroups g{};
  const ObjectState* one = &o;
  make_groups(g, &one, 1);
  LAUNCH(m, st, "assemble_layout", assemble_layout, dim3(m->num_sms * 2, 1), dim3(256), 0, st, (const __half*)nullptr, (const __half*)nullptr,
         t, tab_dev(m), o.xo.hi.as<__half>(), o.xo.lo.as<__half>(), Lo);
  if (int rc = run_gats(m, Lo, o.xo.view(), kPrologueLayer + 0, o.Lf, g, st)) return rc;
  return run_attn_layer(m, Lo, o.xo.view(), kPrologueLayer + 1, m->attn[0], /*cross=*/0, st);
}

// GNN + tail for the `fb` frames of a chunk; frame b matches against fobj[b].  Outputs: m1 / s1 rows and conf rows are M_out wide.
static int forward_chunk(opb_matcher* m, const ObjectState* const* fobj, const float* q_cf, const int* nlen, int N, int fb, int M_out,
                         int64_t* m0, int64_t* m1, float* s0, float* s1, float* conf, cudaStream_t st, int piece, int h2d_first) {
  ChunkTable t{};
  int m_max = 0, m_sum = 0;
  bool uniform = true;
  for (int b = 0; b < fb; ++b) {
    table_frame(t, b, *fobj[b], m->hoist);
    m_max = std::max(m_max, fobj[b]->M);
    m_sum += fobj[b]->M;
    uniform = uniform && fobj[b]->M == fobj[0]->M;
  }
  GatsGroups groups{};
  make_groups(groups, fobj, fb);
  const int Lf = fobj[0]->Lf;
  Layout L{};
  L.B = fb; L.N = N; L.M = m_max; L.n_pad = round_up(N, kSegPad); L.m_pad = round_up(m_max, kSegPad); L.R = L.n_pad + L.m_pad;
  L.nlen = nlen;
  L.mlen = uniform ? nullptr : tab_dev(m)->mlen;     // device address of the table's mlen (written by assemble_layout)
  const int rows = L.rows();
  const double valid_rows = (double)fb * N + m_sum;
  __half *xh = m->x.hi.as<__half>(), *xl = m->x.lo.as<__half>();

  int first_layer = 0;
  if (m->hoist) {
    // layer 1 (self) for the query side only, on a compact [fb*n_pad, 256] buffer; layer 0 does not touch queries.
    // In sub-batches of `piece` frames: with host input (opb_forward_host) each sub-batch starts as soon as ITS descriptors
    // have landed, so the H2D copy of the rest runs under this pass
    for (int p0 = 0, si = 0; p0 < fb; p0 += piece, ++si) {
      const int sb = std::min(piece, fb - p0);
      if (h2d_first + si < m->h2d_pending) CK(m, cudaStreamWaitEvent(st, m->h2d_ev[h2d_first + si], 0));
      Layout Lq{};
      Lq.B = sb; Lq.N = N; Lq.M = 0; Lq.n_pad = L.n_pad; Lq.m_pad = 0; Lq.R = L.n_pad;
      Lq.nlen = nlen ? nlen + p0 : nullptr;
      XView xq = m->xq.view((size_t)p0 * L.n_pad);
      LAUNCH(m, st, "transpose_cf_to_rows", transpose_cf_to_rows<0>, dim3(L.n_pad / 32, sb), dim3(32, 8), 0, st, q_cf + (size_t)p0 * kD * N, N, N,
             (long long)kD * N, Lq.nlen, L.n_pad, xq.hi, xq.lo, (float*)nullptr, (long long)Lq.R, 0);
      m->pass_piece = si;
      const int rc = run_attn_layer(m, Lq, xq, 1, m->attn[0], 0, st);
      m->pass_piece = -1;
      if (rc) return rc;
    }
    // assemble the full layout: query rows from xq, 3D rows from each frame's object prologue
    LAUNCH(m, st, "assemble_layout", assemble_layout, dim3(m->num_sms * 2, fb), dim3(256), 0, st, (const __half*)m->xq.hi.as<__half>(),
           (const __half*)m->xq.lo.as<__half>(), t, tab_dev(m), xh, xl, L);
    first_layer = 2;
  } else {
    // inputs: query descriptors [fb,256,N] channel-first -> q segments; each frame's object rows -> its d segment
    LAUNCH(m, st, "transpose_cf_to_rows", transpose_cf_to_rows<0>, dim3(L.n_pad / 32, fb), dim3(32, 8), 0, st, q_cf, N, N, (long long)kD * N, nlen,
           L.n_pad, xh, xl, (float*)nullptr, (long long)L.R, 0);
    LAUNCH(m, st, "assemble_layout", assemble_layout, dim3(m->num_sms * 2, fb), dim3(256), 0, st, (const __half*)nullptr, (const __half*)nullptr,
           t, tab_dev(m), xh, xl, L);
  }

  for (int layer = first_layer; layer < 12; ++layer) {
    if (layer % 3 == 0) {
      if (int rc = run_gats(m, L, m->x.view(), layer, Lf, groups, st)) return rc;
    } else {
      const int attn_idx = (layer / 3) * 2 + (layer % 3) - 1;
      if (int rc = run_attn_layer(m, L, m->x.view(), layer, m->attn[attn_idx], (layer % 3 == 2) ? 1 : 0, st)) return rc;
    }
  }

  LAUNCH(m, st, "range_check", range_check, dim3((unsigned)(((long long)rows * kD / 8 + 255) / 256)), dim3(256), 0, st, (const __half*)xh,
         (long long)rows * kD / 8, m->range_flag.as<int>());

  // ---- tail (GATs_SuperGlue.py:209-237) ----
  GemmProblem pf{};
  pf.L = L; pf.batch = 1; pf.rows = rows;
  pf.a1 = m->x.c(kD); pf.K1 = kD; pf.b1 = m->wf.c(kD); pf.n_out = 256;
  pf.bias = m->bf.as<float>();
  pf.epi = EPI_L2NORM; pf.out = m->pn.m(kD);       // F.normalize fused into the final_proj epilogue (:209-213)
  if (int rc = gemm(m, pf, st, 2.0 * valid_rows * kD * kD, "final_proj")) return rc;
  if (stop_here(m, kTailLayer, 0, L, m->x.view())) return kStopped;
  // dual softmax + arg-max as two passes of the batched score GEMM (one batch = one frame); the cos matrix is never stored
  const int n_parts = (L.m_pad / 256) * 2, q_groups = L.n_pad / 32;
  GemmProblem ps{};
  ps.L = L; ps.batch = fb; ps.rows = L.n_pad; ps.n_out = L.m_pad;
  ps.a1 = m->pn.c(kD); ps.K1 = kD; ps.b1 = m->pn.c(kD, (size_t)L.n_pad * kD);
  ps.a_batch_rows = L.R; ps.b_batch_rows = L.R;
  ps.inv_scale = 1.f / m->cfg.scale_factor;
  ps.epi = EPI_SCORE_SUMS; ps.rowsum_part = m->rowsum_part.as<float>(); ps.colsum_part = m->colsum_part.as<float>();
  if (int rc = gemm(m, ps, st, 2.0 * (double)N * m_sum * kD, "score_sums")) return rc;
  if (stop_here(m, kTailLayer, 1, L, m->x.view())) return kStopped;
  LAUNCH(m, st, "score_sums_finalize", score_sums_finalize, dim3((L.n_pad + L.m_pad + 255) / 256, fb), dim3(256), 0, st,
         (const float*)m->rowsum_part.as<float>(), (const float*)m->colsum_part.as<float>(), L, n_parts, q_groups, m->rowsum.as<float>(),
         m->colsum.as<float>(), m->rowbest.as<unsigned long long>(), m->colbest.as<unsigned long long>());
  if (stop_here(m, kTailLayer, 2, L, m->x.view())) return kStopped;
  ps.epi = EPI_SCORE_CONF; ps.inv_rowsum = m->rowsum.as<float>(); ps.inv_colsum = m->colsum.as<float>();
  ps.conf = conf; ps.conf_ld = M_out; ps.rowbest = m->rowbest.as<unsigned long long>(); ps.colbest = m->colbest.as<unsigned long long>();
  if (int rc = gemm(m, ps, st, 0.0, "score_conf")) return rc;      // recomputation: its FLOPs are not algorithmic
  if (stop_here(m, kTailLayer, 3, L, m->x.view())) return kStopped;
  if (conf && M_out > L.m_pad)                                          // conf rows wider than this chunk's 3D segments
    LAUNCH(m, st, "conf_fill_tail", conf_fill_tail, dim3(m->num_sms * 4), dim3(256), 0, st, conf, (long long)fb * N, M_out, L.m_pad);
  LAUNCH(m, st, "mutual_match", mutual_match, dim3(fb), dim3(256), 0, st, (const unsigned long long*)m->rowbest.as<unsigned long long>(),
         (const unsigned long long*)m->colbest.as<unsigned long long>(), L, m->cfg.match_threshold, (const int*)m->range_flag.as<int>(), M_out,
         reinterpret_cast<long long*>(m0), reinterpret_cast<long long*>(m1), s0, s1);
  return 0;
}

static int chunk_of(const opb_matcher* m, int B) {
  int chunk = m->chunk_frames > 0 ? m->chunk_frames : kDefaultChunk;
  return chunk > B ? B : chunk;
}

// Leaf logits of an object (frame-invariant, they depend on the weights): GATs.py:40,78 folded as s2 = leaves . (W a[:256]).
// Not counted here: it also runs outside a forward (opb_set_object / opb_add_object), where it must not touch the profile of
// the last forward; forward_frames counts it.
static cudaError_t launch_leaf_logits(const opb_matcher* m, const ObjectState& o, cudaStream_t st) {
  return launch_k(pdl_enabled(), gats_leaf_logits, dim3(m->num_sms * 4), dim3(256), 0, st, (const float*)o.leaves.as<float>(),
                  (long long)o.M * o.Lf, (const float*)m->wa2.as<float>(), o.s2.as<float>());
}

// Upload an object's constants into `o` (buffers only grow) and compute its leaf logits; its prologue runs on first use.
static int load_object(opb_matcher* m, ObjectState& o, const float* desc3d_db, const float* desc2d_db, int M, int Lf, cudaStream_t st) {
  const int m_pad = round_up(M, kSegPad);
  o.M = M; o.Lf = Lf; o.m_pad = m_pad;
  const long long n_leaf_rows = (long long)M * Lf;
  o.leaves.grew = o.db.hi.grew = o.s2.grew = o.xo.hi.grew = false;
  o.s2_ready = o.prologue_ready = false;
  CK(m, o.leaves.ensure((size_t)n_leaf_rows * kD * sizeof(float)));
  CK(m, o.db.ensure((size_t)m_pad * kD));
  CK(m, o.s2.ensure((size_t)4 * n_leaf_rows * sizeof(float)));
  CK(m, o.xo.ensure((size_t)m_pad * kD));
  if (o.leaves.grew || o.db.hi.grew || o.s2.grew || o.xo.hi.grew) CK(m, cudaDeviceSynchronize());   // frees of the old buffers vs work in flight
  launch_k(pdl_enabled(), transpose_cf_to_rows<1>, dim3((unsigned)((n_leaf_rows + 31) / 32), 1), dim3(32, 8), 0, st, desc2d_db, (int)n_leaf_rows,
           (int)n_leaf_rows, 0ll, (const int*)nullptr, (int)n_leaf_rows, (__half*)nullptr, (__half*)nullptr, o.leaves.as<float>(), 0ll, 0);
  // rows [M, m_pad) of the object planes are written as zero by the transpose (MODE 0 pads to rows_out)
  launch_k(pdl_enabled(), transpose_cf_to_rows<0>, dim3(m_pad / 32, 1), dim3(32, 8), 0, st, desc3d_db, (int)M, (int)M, 0ll, (const int*)nullptr,
           m_pad, o.db.hi.as<__half>(), o.db.lo.as<__half>(), (float*)nullptr, 0ll, 0);
  CK(m, cudaGetLastError());
  CK(m, launch_leaf_logits(m, o, st));
  o.s2_ready = true;
  return 0;
}

// opb_set_object / opb_add_object (`fn`; `need`: its argument conditions; `id_ok`: false for a null id pointer): loads an object
// into the entry under `key`, reusing the buffers of an entry already there.  A failed load leaves no entry under `key`.
static int load_entry(opb_matcher* m, const char* fn, const char* need, int key, const float* desc3d_db, const float* desc2d_db, int M, int Lf,
                      bool id_ok, cudaStream_t st) {
  if (!m->weights_ready) return fail(m, OPB_E_STATE, "opb_%s before opb_finalize_weights", fn);
  if (!desc3d_db || !desc2d_db || !id_ok || M <= 0 || Lf <= 0 || Lf > 32)
    return fail(m, OPB_E_INVALID, "%s: need %s (got M=%d, L=%d)", fn, need, M, Lf);
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  ObjectState& o = m->objects[key];
  if (int rc = ordered(m, st, [&] { return load_object(m, o, desc3d_db, desc2d_db, M, Lf, st); })) {
    cudaDeviceSynchronize();                       // work in flight may still read the entry's buffers
    m->objects.erase(key);
    return rc;
  }
  return OPB_OK;
}

static ObjectState* find_object(opb_matcher* m, int key) { return m->objects.count(key) ? &m->objects.at(key) : nullptr; }

// An object of opb_add_object by the id a caller passed: no such id reaches the current object's reserved key.
static ObjectState* registered(opb_matcher* m, int id) { return id == kCurrentObject ? nullptr : find_object(m, id); }

static void invalidate_prologues(opb_matcher* m) {
  for (auto& kv : m->objects) kv.second.prologue_ready = false;
}

// A forward that reached the stop of opb_debug_set_stop: its buffers stay as they are for opb_debug_read.
static int stopped(opb_matcher* m, cudaStream_t st) {
  m->timeline.finish(st);
  m->last_launches = m->launches;
  return OPB_OK;
}

// The one forward of the handle: frame b of the call matches against fobj[b] (opb_forward: the current object everywhere).
// m1 / s1 rows and conf rows are M_out >= max M_b wide.
static int forward_frames(opb_matcher* m, ObjectState* const* fobj, const float* q, const int32_t* n2d_lengths, int B, int N, int M_out,
                          int64_t* m0, int64_t* m1, float* s0, float* s1, float* conf, cudaStream_t st) {
  int call_m_pad = 0;
  for (int b = 0; b < B; ++b) call_m_pad = std::max(call_m_pad, fobj[b]->m_pad);
  const int chunk = chunk_of(m, B);
  if (int rc = ensure_workspace(m, chunk, N, call_m_pad)) return rc;   // no-op once opb_reserve_workspace / an earlier call has sized it
  m->begin(st);
  m->dbg_stopped = false;
  // per-object work on first use: leaf logits after a weight reload, the prologue (once per object, shared by all later calls)
  for (int b = 0; b < B; ++b) {
    ObjectState& o = *fobj[b];
    if (!o.s2_ready) {
      if (int rc = launched(m, st, "gats_leaf_logits", launch_leaf_logits(m, o, st))) return rc;
      o.s2_ready = true;
    }
    if (m->hoist && !o.prologue_ready) {
      if (int rc = object_prologue(m, o, st)) return rc == kStopped ? stopped(m, st) : rc;
      o.prologue_ready = true;
    }
  }
  // granularity of the query-side layer-1 pass: the host-copy pieces when the queries stream in from the host, else the chunk
  const int piece = m->h2d_pending > 0 ? std::min(chunk, kQPassFrames) : chunk;
  const int ppc = (chunk + piece - 1) / piece;              // pieces per chunk
  for (int f0 = 0, ci = 0; f0 < B; f0 += chunk, ++ci) {
    const int fb = std::min(chunk, B - f0);
    if (!m->hoist)                                          // per-frame evaluation consumes the whole chunk at once
      for (int si = 0; si * piece < fb; ++si)
        if (ci * ppc + si < m->h2d_pending) CK(m, cudaStreamWaitEvent(st, m->h2d_ev[ci * ppc + si], 0));
    m->pass_chunk = ci;
    int rc = forward_chunk(m, fobj + f0, q + (size_t)f0 * kD * N, n2d_lengths ? n2d_lengths + f0 : nullptr, N, fb, M_out, m0 + (size_t)f0 * N,
                           m1 + (size_t)f0 * M_out, s0 + (size_t)f0 * N, s1 + (size_t)f0 * M_out, conf ? conf + (size_t)f0 * N * M_out : nullptr,
                           st, piece, ci * ppc);
    if (rc) return rc == kStopped ? stopped(m, st) : rc;
  }
  // deferred range report: the flag travels to pinned host memory behind the call (current once the handle's event, recorded
  // behind it, has completed); opb_poll_range() reads it without blocking
  CK(m, cudaMemcpyAsync(m->range_host, m->range_flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  m->range_pending = true;
  m->timeline.finish(st);
  m->last_launches = m->launches;
  return OPB_OK;
}

// A segmented mean: the offsets (exclusive scan of seg_len) in a stream-ordered temporary, then segmented_mean_f64; the
// temporary is freed behind it whether or not the launches succeed.
static int segmented(const char* fn, const double* x, const int64_t* seg_len, int32_t M, int32_t D, int channel_major, double* out,
                     cudaStream_t st) {
  const long long* len = reinterpret_cast<const long long*>(seg_len);
  long long* offs = nullptr;
  CK(no_handle_error, cudaMallocAsync(&offs, (size_t)M * sizeof(long long), st));
  const unsigned grid = (unsigned)std::min<long long>(((long long)M * D + 255) / 256, 1 << 20);   // grid-stride past 2^28 entries
  int rc = launched(fn, "exclusive_scan_i64", launch_k(false, exclusive_scan_i64, 1, 1024, 0, st, len, offs, M));
  if (rc == OPB_OK)
    rc = launched(fn, "segmented_mean_f64", launch_k(false, segmented_mean_f64, grid, 256, 0, st, x, len, offs, M, D, channel_major, out));
  CK(no_handle_error, cudaFreeAsync(offs, st));
  return rc;
}

// opb_debug_block's kernels: one block walks `tiles` tiles of blockDim.x inputs and calls one primitive of block.cuh per tile,
// always with the same sh, as the library's tile loops do.  Per thread and tile: what the primitive returned, and the total.
template <typename T, typename Op>
__global__ void debug_block_scan(int prim, Op op, T identity, bool reverse, int tiles, const T* __restrict__ in, T* __restrict__ value,
                                 T* __restrict__ total) {
  __shared__ T sh[32];
  for (int t = 0; t < tiles; ++t) {
    const size_t i = (size_t)t * blockDim.x + threadIdx.x;
    T all;
    const T v = prim == 0 ? (all = block_reduce(in[i], op, sh)) : block_scan(in[i], op, identity, sh, &all, reverse);
    value[i] = v;
    total[i] = all;
  }
}

__global__ void debug_block_rank(int tiles, const int32_t* __restrict__ keep, int32_t* __restrict__ value, int32_t* __restrict__ total) {
  __shared__ int sh[32];
  for (int t = 0; t < tiles; ++t) {
    const size_t i = (size_t)t * blockDim.x + threadIdx.x;
    int all;
    value[i] = block_rank(keep[i] != 0, sh, &all);
    total[i] = all;
  }
}

template <typename T, typename Op>
static int debug_block_launch(int prim, Op op, T identity, bool reverse, int threads, int tiles, const void* in, void* value, void* total,
                              cudaStream_t st) {
  return launched("opb_debug_block", "debug_block_scan",
                  launch_k(false, debug_block_scan<T, Op>, 1, threads, 0, st, prim, op, identity, reverse, tiles, (const T*)in, (T*)value, (T*)total));
}

}  // namespace opb

// =========================================================================================
extern "C" {

int opb_create(const opb_config* cfg, opb_matcher** out) {
  if (!cfg || !out) return fail(no_handle_error, OPB_E_INVALID, "null argument");
  if (cfg->descriptor_dim != kD || cfg->num_heads != kHeads)
    return fail(no_handle_error, OPB_E_INVALID, "only descriptor_dim=256, num_heads=4 are supported (got %d, %d)", cfg->descriptor_dim,
                cfg->num_heads);
  // The tail's fixed shift e = exp((cos - 1) / scale) runs on ex2.approx.ftz, which flushes results below 2^-126 to zero: every
  // cosine in [-1, 1] keeps e a normal fp32 value only when 2 log2(e) / scale <= 126.  Below that a query whose cosines are all
  // low would get a zero row sum and a NaN conf row.
  if (!((double)cfg->scale_factor >= kMinScaleFactor))
    return fail(no_handle_error, OPB_E_INVALID, "scale_factor must be >= 2 log2(e) / 126 = %.6f (got %g)", kMinScaleFactor, (double)cfg->scale_factor);
  cudaDeviceProp prop;
  if (int rc = select_device(cfg->device, prop, no_handle_error)) return rc;
  DeviceGuard dg(cfg->device);
  if (dg.err) return fail(no_handle_error, OPB_E_CUDA, "cudaSetDevice: %s", cudaGetErrorString(dg.err));
  auto* m = new opb_matcher();
  m->cfg = *cfg;
  m->num_sms = prop.multiProcessorCount;
  if (int rc = create_handle_state(m, cfg->device, &m->range_host, no_handle_error)) {
    delete m;
    return rc;
  }
  *out = m;
  return OPB_OK;
}

void opb_destroy(opb_matcher* m) {
  if (!m) return;
  DeviceGuard dg(m->device);
  cudaDeviceSynchronize();   // the frees of the handle's buffers come after the work in flight
  delete m;
}

const char* opb_last_error(const opb_matcher* m) { return m ? m->err.c_str() : no_handle_error.c_str(); }

int opb_load_weight(opb_matcher* m, const char* name, const float* data, size_t n) {
  if (!m || !name || !data) return m ? fail(m, OPB_E_INVALID, "null argument") : fail(no_handle_error, OPB_E_INVALID, "null argument");
  m->host_w[name] = std::vector<float>(data, data + n);
  m->weights_ready = false;
  return OPB_OK;
}

int opb_finalize_weights(opb_matcher* m) {
  if (!m) return OPB_E_INVALID;
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  CK(m, m->drain());          // the uploads below are host copies: calls in flight may still read the old weights
  // head-contiguous channel order: new c' = h*64 + d  <-  reference c = d*4 + h (GATs_SuperGlue.py:97)
  int perm[kD];
  for (int h = 0; h < kHeads; ++h)
    for (int d = 0; d < kDh; ++d) perm[h * kDh + d] = d * kHeads + h;
  std::vector<double> wa2(4 * kD), wa3(4 * kD);
  int ai = 0;
  for (int layer = 0; layer < 12; ++layer) {
    const std::string p = "gnn.layers." + std::to_string(layer);
    if (layer % 3 == 0) {
      auto* W = find_weight(m, p + ".W", kD * kD);
      auto* a = find_weight(m, p + ".a", 2 * kD);
      if (!W || !a) return m->find_code;
      const int gi = layer / 3;
      for (int c = 0; c < kD; ++c) {  // h @ W @ a[:256] = h . (W a[:256])   (GATs.py:40,78-80)
        double s2 = 0, s3 = 0;
        for (int o = 0; o < kD; ++o) {
          s2 += (double)(*W)[c * kD + o] * (double)(*a)[o];
          s3 += (double)(*W)[c * kD + o] * (double)(*a)[kD + o];
        }
        wa2[gi * kD + c] = s2;
        wa3[gi * kD + c] = s3;
      }
      if (m->cfg.with_linear_transform) {     // B operand of  t = pre . W :  B[o][c] = W[c][o]
        std::vector<double> wt((size_t)kD * kD);
        for (int c = 0; c < kD; ++c)
          for (int o = 0; o < kD; ++o) wt[(size_t)o * kD + c] = (*W)[(size_t)c * kD + o];
        if (int rc = upload_planes(m, m->wlin, wt, (size_t)gi * kD * kD, (size_t)4 * kD * kD)) return rc;
      }
      continue;
    }
    AttnLayerW& A = m->attn[ai++];
    const std::vector<float>*Wp[3], *bp[3];
    for (int j = 0; j < 3; ++j) {
      Wp[j] = find_weight(m, p + ".attn.proj." + std::to_string(j) + ".weight", kD * kD);
      bp[j] = find_weight(m, p + ".attn.proj." + std::to_string(j) + ".bias", kD);
      if (!Wp[j] || !bp[j]) return m->find_code;
    }
    auto* Wm = find_weight(m, p + ".attn.merge.weight", kD * kD);
    auto* bm = find_weight(m, p + ".attn.merge.bias", kD);
    auto* W0 = find_weight(m, p + ".mlp.0.weight", 512 * 512);
    auto* b0 = find_weight(m, p + ".mlp.0.bias", 512);
    auto* W1 = find_weight(m, p + ".mlp.3.weight", kD * 512);
    auto* b1 = find_weight(m, p + ".mlp.3.bias", kD);
    if (!Wm || !bm || !W0 || !b0 || !W1 || !b1) return m->find_code;
    std::vector<double> wqkv(768 * kD), bqkv(768);
    for (int j = 0; j < 3; ++j)
      for (int c = 0; c < kD; ++c) {
        for (int k = 0; k < kD; ++k) wqkv[((size_t)j * kD + c) * kD + k] = (*Wp[j])[(size_t)perm[c] * kD + k];
        bqkv[j * kD + c] = (*bp[j])[perm[c]];
      }
    std::vector<double> w0a(512 * kD), w0m(512 * kD), b0f(512);
    for (int c = 0; c < 512; ++c) {
      for (int k = 0; k < kD; ++k) w0a[(size_t)c * kD + k] = (*W0)[(size_t)c * 512 + k];
      double bacc = (*b0)[c];
      for (int o = 0; o < kD; ++o) bacc += (double)(*W0)[(size_t)c * 512 + kD + o] * (double)(*bm)[o];
      b0f[c] = bacc;
      for (int k = 0; k < kD; ++k) {  // message channel k (head-contiguous) = reference channel perm[k]
        double acc = 0;
        for (int o = 0; o < kD; ++o) acc += (double)(*W0)[(size_t)c * 512 + kD + o] * (double)(*Wm)[(size_t)o * kD + perm[k]];
        w0m[(size_t)c * kD + k] = acc;
      }
    }
    std::vector<double> w1(W1->begin(), W1->end()), b1d(b1->begin(), b1->end());
    if (int rc = upload_planes(m, A.wqkv, wqkv)) return rc;
    if (int rc = upload_f32(m, A.bqkv, bqkv)) return rc;
    if (int rc = upload_planes(m, A.w0a, w0a)) return rc;
    if (int rc = upload_planes(m, A.w0m, w0m)) return rc;
    if (int rc = upload_f32(m, A.b0f, b0f)) return rc;
    if (int rc = upload_planes(m, A.w1, w1)) return rc;
    if (int rc = upload_f32(m, A.b1, b1d)) return rc;
  }
  auto* Wf = find_weight(m, "final_proj.weight", kD * kD);
  auto* bfv = find_weight(m, "final_proj.bias", kD);
  if (!Wf || !bfv) return m->find_code;
  if (int rc = upload_planes(m, m->wf, std::vector<double>(Wf->begin(), Wf->end()))) return rc;
  {
    std::vector<double> eye((size_t)kD * kD, 0.0);
    for (int i = 0; i < kD; ++i) eye[(size_t)i * kD + i] = 1.0;
    if (int rc = upload_planes(m, m->eye, eye)) return rc;
  }
  if (int rc = upload_f32(m, m->bf, std::vector<double>(bfv->begin(), bfv->end()))) return rc;
  if (int rc = upload_f32(m, m->wa2, wa2)) return rc;
  if (int rc = upload_f32(m, m->wa3, wa3)) return rc;
  CK(m, cudaDeviceSynchronize());
  m->weights_ready = true;
  m->objects.erase(kCurrentObject);   // s2 and the prologue depend on the weights: the current object is set again, registered
  for (auto& kv : m->objects) kv.second.s2_ready = kv.second.prologue_ready = false;   // objects recompute theirs on their next use
  return OPB_OK;
}

int opb_set_object(opb_matcher* m, const float* desc3d_db, const float* desc2d_db, int32_t M, int32_t Lf, void* stream) {
  if (!m) return OPB_E_INVALID;
  return load_entry(m, "set_object", "M > 0 and 1 <= num_leaf <= 32", kCurrentObject, desc3d_db, desc2d_db, M, Lf, /*id_ok=*/true, (cudaStream_t)stream);
}

int opb_add_object(opb_matcher* m, const float* desc3d_db, const float* desc2d_db, int32_t M, int32_t Lf, void* stream, int32_t* object_id) {
  if (!m) return OPB_E_INVALID;
  const int rc = load_entry(m, "add_object", "M > 0, 1 <= num_leaf <= 32 and an id pointer", m->next_object_id, desc3d_db, desc2d_db, M, Lf,
                            object_id != nullptr, (cudaStream_t)stream);
  if (rc == OPB_OK) *object_id = m->next_object_id++;
  return rc;
}

int opb_remove_object(opb_matcher* m, int32_t object_id) {
  if (!m) return OPB_E_INVALID;
  if (!registered(m, object_id)) return fail(m, OPB_E_INVALID, "remove_object: unknown object id %d", object_id);
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  CK(m, cudaDeviceSynchronize());                  // calls in flight may still read the object's buffers
  m->objects.erase(object_id);
  return OPB_OK;
}

int opb_reserve_workspace(opb_matcher* m, int32_t frames, int32_t N) {
  if (!m || frames <= 0 || N <= 0) return OPB_E_INVALID;
  if (m->objects.empty()) return fail(m, OPB_E_STATE, "opb_reserve_workspace needs an object (the workspace depends on M)");
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  int m_pad = 0;                                   // sized for the largest object the handle knows
  for (auto& kv : m->objects) m_pad = std::max(m_pad, kv.second.m_pad);
  return ensure_workspace(m, chunk_of(m, frames), N, m_pad);
}

int opb_set_hoist(opb_matcher* m, int32_t enable) {
  if (!m) return OPB_E_INVALID;
  m->hoist = enable != 0;
  return OPB_OK;
}

int opb_set_chunk_frames(opb_matcher* m, int32_t frames) {
  if (!m || frames < 0) return OPB_E_INVALID;
  if (frames > kMaxChunkFrames)            // the per-chunk object table (ChunkTable) is a kernel parameter of fixed size
    return fail(m, OPB_E_INVALID, "opb_set_chunk_frames: at most %d frames per chunk (got %d)", kMaxChunkFrames, frames);
  m->chunk_frames = frames;
  return OPB_OK;
}

int opb_forward(opb_matcher* m, const float* q, const int32_t* n2d_lengths, int32_t B, int32_t N, int64_t* m0, int64_t* m1, float* s0, float* s1,
                float* conf, void* stream) {
  if (!m) return OPB_E_INVALID;
  ObjectState* cur = find_object(m, kCurrentObject);
  if (!m->weights_ready || !cur) return fail(m, OPB_E_STATE, "opb_forward needs weights and an object (finalize_weights, set_object)");
  if (!q || !m0 || !m1 || !s0 || !s1 || B <= 0 || N <= 0) return fail(m, OPB_E_INVALID, "opb_forward: bad argument (B=%d, N=%d)", B, N);
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  const cudaStream_t st = (cudaStream_t)stream;
  std::vector<ObjectState*> fobj((size_t)B, cur);           // every frame uses the current object
  return ordered(m, st, [&] { return forward_frames(m, fobj.data(), q, n2d_lengths, B, N, cur->M, m0, m1, s0, s1, conf, st); });
}

int opb_forward_objects(opb_matcher* m, const int32_t* object_ids_host, const float* q, const int32_t* n2d_lengths, int32_t B, int32_t N,
                        int32_t M_out, int64_t* m0, int64_t* m1, float* s0, float* s1, float* conf, void* stream) {
  if (!m) return OPB_E_INVALID;
  if (!m->weights_ready) return fail(m, OPB_E_STATE, "opb_forward_objects needs weights (finalize_weights)");
  if (!object_ids_host || !q || !m0 || !m1 || !s0 || !s1 || B <= 0 || N <= 0)
    return fail(m, OPB_E_INVALID, "opb_forward_objects: bad argument (B=%d, N=%d)", B, N);
  std::vector<ObjectState*> fobj((size_t)B);
  int m_max = 0;
  for (int b = 0; b < B; ++b) {
    fobj[b] = registered(m, object_ids_host[b]);
    if (!fobj[b]) return fail(m, OPB_E_INVALID, "opb_forward_objects: unknown object id %d (frame %d)", object_ids_host[b], b);
    if (fobj[b]->Lf != fobj[0]->Lf)
      return fail(m, OPB_E_INVALID, "opb_forward_objects: frames %d and 0 use objects with different leaf counts (%d, %d)", b, fobj[b]->Lf,
                  fobj[0]->Lf);
    m_max = std::max(m_max, fobj[b]->M);
  }
  if (M_out < m_max) return fail(m, OPB_E_INVALID, "opb_forward_objects: M_out = %d is below the largest object of the call (M = %d)", M_out, m_max);
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  const cudaStream_t st = (cudaStream_t)stream;
  return ordered(m, st, [&] { return forward_frames(m, fobj.data(), q, n2d_lengths, B, N, M_out, m0, m1, s0, s1, conf, st); });
}

int opb_set_profiling(opb_matcher* m, int32_t enable) {
  if (!m) return OPB_E_INVALID;
  m->timeline.on = enable != 0;
  m->timeline.clear();
  return OPB_OK;
}

int opb_get_profile(opb_matcher* m, double* gemm_ms, double* gemm_flops, int32_t* gemm_launches, double* total_ms) {
  if (!m || !m->timeline.end) return OPB_E_STATE;
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  const Timeline& tl = m->timeline;
  CK(m, cudaEventSynchronize(tl.end));
  double ms = 0, fl = 0;
  int n_gemm = 0;
  std::map<std::string, std::pair<double, std::pair<double, int>>> agg;
  for (size_t i = 0; i < tl.size(); ++i) {
    float t = 0;
    CK(m, tl.ms(i, &t));
    if (tl.name[i].compare(0, 4, "gemm") == 0) { ms += t; fl += tl.flops[i]; ++n_gemm; }
    auto& a = agg[tl.name[i]];
    a.first += t; a.second.first += tl.flops[i]; a.second.second++;
  }
  float tot = 0;
  CK(m, cudaEventElapsedTime(&tot, tl.start, tl.end));
  if (getenv("OPB_PROFILE_DUMP")) {   // measurement aid only: prints the table, selects nothing
    fprintf(stderr, "[opb profile] forward %.3f ms, GEMM %.3f ms in %d launches\n", tot, ms, n_gemm);
    for (auto& kv : agg)
      fprintf(stderr, "[opb profile] %-36s %4d launches %8.3f ms %5.1f%%  %7.1f TFLOP/s algorithmic\n", kv.first.c_str(), kv.second.second.second,
              kv.second.first, 100.0 * kv.second.first / tot, kv.second.second.first / (kv.second.first * 1e-3) / 1e12);
  }
  if (gemm_ms) *gemm_ms = ms;
  if (gemm_flops) *gemm_flops = fl;
  if (gemm_launches) *gemm_launches = (int32_t)n_gemm;
  if (total_ms) *total_ms = tot;
  return OPB_OK;
}

int opb_get_profile_entry(opb_matcher* m, const char* prefix, double* ms_out, double* flops_out, int32_t* launches_out) {
  if (!m || !prefix || !m->timeline.end) return OPB_E_STATE;
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  const Timeline& tl = m->timeline;
  CK(m, cudaEventSynchronize(tl.end));
  double ms = 0, fl = 0;
  int n = 0;
  const size_t pl = strlen(prefix);
  for (size_t i = 0; i < tl.size(); ++i) {
    if (tl.name[i].compare(0, pl, prefix) != 0) continue;
    float t = 0;
    CK(m, tl.ms(i, &t));
    ms += t; fl += tl.flops[i]; ++n;
  }
  if (ms_out) *ms_out = ms;
  if (flops_out) *flops_out = fl;
  if (launches_out) *launches_out = n;
  return OPB_OK;
}

int opb_forward_host(opb_matcher* m, const float* qh, const int32_t* n2d_lengths_host, int32_t B, int32_t N, int64_t* m0h, int64_t* m1h, float* s0h,
                     float* s1h, float* confh, int32_t materialize_conf, void* stream) {
  if (!m) return OPB_E_INVALID;
  const ObjectState* cur = find_object(m, kCurrentObject);
  if (!cur) return fail(m, OPB_E_STATE, "opb_forward_host needs an object");
  if (!qh || !m0h || !m1h || !s0h || !s1h || B <= 0 || N <= 0) return fail(m, OPB_E_INVALID, "opb_forward_host: bad argument");
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t M = cur->M;
  const bool want_conf = confh != nullptr || materialize_conf != 0;
  DevBuf* stg[] = {&m->st_q, &m->st_m0, &m->st_m1, &m->st_s0, &m->st_s1, &m->st_conf, &m->st_len};
  for (auto* b : stg) b->grew = false;
  CK(m, m->st_q.ensure((size_t)B * kD * N * sizeof(float)));
  CK(m, m->st_m0.ensure((size_t)B * N * sizeof(int64_t)));
  CK(m, m->st_m1.ensure((size_t)B * M * sizeof(int64_t)));
  CK(m, m->st_s0.ensure((size_t)B * N * sizeof(float)));
  CK(m, m->st_s1.ensure((size_t)B * M * sizeof(float)));
  if (want_conf) CK(m, m->st_conf.ensure((size_t)B * N * M * sizeof(float)));
  if (n2d_lengths_host) CK(m, m->st_len.ensure((size_t)B * sizeof(int32_t)));
  // H2D per piece on a side stream: the copy of piece i+1 runs under the compute of piece i
  const int chunk = chunk_of(m, B);
  if (!m->copy_stream) CK(m, cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
  const int piece = std::min(chunk, kQPassFrames);
  const int ppc = (chunk + piece - 1) / piece;
  const int n_chunks = (B + chunk - 1) / chunk;
  const int n_ev = n_chunks * ppc;
  while ((int)m->h2d_ev.size() < n_ev + 1) {
    cudaEvent_t e;
    CK(m, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    m->h2d_ev.push_back(e);
  }
  const int rc = ordered(m, st, [&] {
    CK(m, cudaEventRecord(m->h2d_ev[n_ev], st));                         // staging buffer reuse: wait for earlier work on `st`
    CK(m, cudaStreamWaitEvent(m->copy_stream, m->h2d_ev[n_ev], 0));
    if (n2d_lengths_host) CK(m, cudaMemcpyAsync(m->st_len.p, n2d_lengths_host, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, m->copy_stream));
    for (int ci = 0; ci < n_chunks; ++ci) {
      const int c0 = ci * chunk, cb = std::min(chunk, B - c0);
      for (int si = 0; si < ppc; ++si) {
        const int f0 = c0 + si * piece, fb = std::min(piece, c0 + cb - f0);
        if (fb > 0) {
          const size_t off = (size_t)f0 * kD * N;
          CK(m, cudaMemcpyAsync(m->st_q.as<float>() + off, qh + off, (size_t)fb * kD * N * sizeof(float), cudaMemcpyHostToDevice, m->copy_stream));
        }
        CK(m, cudaEventRecord(m->h2d_ev[ci * ppc + si], m->copy_stream));
      }
    }
    m->h2d_pending = n_ev;
    const int frc = opb_forward(m, m->st_q.as<float>(), n2d_lengths_host ? m->st_len.as<int32_t>() : nullptr, B, N, m->st_m0.as<int64_t>(),
                                m->st_m1.as<int64_t>(), m->st_s0.as<float>(), m->st_s1.as<float>(), want_conf ? m->st_conf.as<float>() : nullptr, stream);
    m->h2d_pending = 0;
    if (frc) return frc;
    CK(m, cudaMemcpyAsync(m0h, m->st_m0.p, (size_t)B * N * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CK(m, cudaMemcpyAsync(m1h, m->st_m1.p, (size_t)B * M * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CK(m, cudaMemcpyAsync(s0h, m->st_s0.p, (size_t)B * N * sizeof(float), cudaMemcpyDeviceToHost, st));
    CK(m, cudaMemcpyAsync(s1h, m->st_s1.p, (size_t)B * M * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (confh) CK(m, cudaMemcpyAsync(confh, m->st_conf.p, (size_t)B * N * M * sizeof(float), cudaMemcpyDeviceToHost, st));
    return (int)OPB_OK;
  });
  if (rc) return rc;
  CK(m, cudaStreamSynchronize(st));
  return opb_check_range(m, stream);
}

// Consume the range flag.  Once the handle's event has completed, the pinned copy written behind the last opb_forward is
// current.  The reset of the device flag is a call of the handle like any other: the next call, on whatever stream, comes after it.
static int consume_range_flag(opb_matcher* m) {
  m->range_pending = false;
  if (*m->range_host == 0) return OPB_OK;
  *m->range_host = 0;
  const cudaStream_t st = m->ev_stream;
  if (int rc = ordered(m, st, [&] {
        CK(m, cudaMemsetAsync(m->range_flag.p, 0, sizeof(int), st));
        return (int)OPB_OK;
      }))
    return rc;
  return fail(m, OPB_E_RANGE, "an activation left the fp16-split operand range (|x| >= 1023) or became NaN: the matches of that call were "
                              "reported as -1 (no match)");
}

int opb_check_range(opb_matcher* m, void* stream) {
  if (!m || !m->range_flag.p || !m->range_pending) return OPB_OK;
  (void)stream;
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  CK(m, cudaEventSynchronize(m->ev));
  return consume_range_flag(m);
}

int opb_poll_range(opb_matcher* m) {
  if (!m || !m->range_pending) return OPB_OK;
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  const cudaError_t q = cudaEventQuery(m->ev);
  if (q == cudaErrorNotReady) return OPB_OK;               // the call is still running: report on a later poll / check
  if (q != cudaSuccess) return fail(m, OPB_E_CUDA, "cudaEventQuery: %s", cudaGetErrorString(q));
  return consume_range_flag(m);
}

int opb_last_launch_count(const opb_matcher* m) { return m ? m->last_launches : 0; }

// ---- adjacent producers ------------------------------------------------------------------
int opb_segmented_mean_f64(const double* desc, const int64_t* seg_len, int32_t M, int32_t D, double* out, void* stream) {
  REQUIRE(__func__, desc && seg_len && out && M > 0 && D > 0);
  return segmented(__func__, desc, seg_len, M, D, 0, out, (cudaStream_t)stream);
}

int opb_segmented_mean_channels_f64(const double* desc, const int64_t* seg_len, int32_t M, int32_t D, double* out, void* stream) {
  REQUIRE(__func__, desc && seg_len && out && M > 0 && D > 0);
  return segmented(__func__, desc, seg_len, M, D, 1, out, (cudaStream_t)stream);
}

int opb_segmented_mean_scores_f64(const double* scores, const int64_t* seg_len, int32_t M, double* out, void* stream) {
  REQUIRE(__func__, scores && seg_len && out && M > 0);
  return segmented(__func__, scores, seg_len, M, 1, 1, out, (cudaStream_t)stream);
}

int opb_gather_features3d(const float* desc, const float* scores, int32_t dim, int64_t n_src, const int64_t* idx, int64_t n_idx, float* desc_out,
                          float* scores_out, int64_t n_out, void* stream) {
  REQUIRE(__func__, (desc || n_src == 0) && (desc_out || n_out == 0) && dim > 0 && dim <= 65535 && n_src >= 0 && n_out >= 0 && n_idx >= 0 &&
                        n_idx <= n_out);   // dim is gridDim.y
  if (n_out == 0) return OPB_OK;                           // n_target_shape = 0: empty outputs, as the reference gives
  cudaStream_t st = (cudaStream_t)stream;
  const unsigned gx = (unsigned)((n_out + 255) / 256);
  LAUNCH_NH(__func__, gather_columns_f32, dim3(gx, (unsigned)dim), 256, 0, st, desc, dim, (long long)n_src, reinterpret_cast<const long long*>(idx),
            (long long)n_idx, desc_out, (long long)n_out);
  if (scores_out && (scores || n_src == 0))                // no source scores: every output score is dustbin or padding
    LAUNCH_NH(__func__, gather_scores_f32, gx, 256, 0, st, scores, (long long)n_src, reinterpret_cast<const long long*>(idx), (long long)n_idx,
              scores_out, (long long)n_out);
  return OPB_OK;
}

// ---- test hooks ---------------------------------------------------------------------------
int opb_debug_set_kv_passes(opb_matcher* m, int32_t passes) {
  if (!m || (passes != 2 && passes != 3)) return OPB_E_INVALID;
  m->kv_two_pass = passes == 2 ? 1 : 0;
  invalidate_prologues(m);
  return OPB_OK;
}

int opb_debug_set_stop(opb_matcher* m, int32_t layer, int32_t step) {
  if (!m || layer < -1 || step < 0) return OPB_E_INVALID;
  m->dbg_layer = layer;
  m->dbg_step = step;
  return OPB_OK;
}

int opb_debug_invalidate_prologues(opb_matcher* m) {
  if (!m) return OPB_E_INVALID;
  invalidate_prologues(m);
  return OPB_OK;
}

int opb_debug_set_stop_pass(opb_matcher* m, int32_t chunk, int32_t piece) {
  if (!m || chunk < 0 || piece < 0) return OPB_E_INVALID;
  m->dbg_chunk = chunk;
  m->dbg_piece = piece;
  return OPB_OK;
}

int opb_debug_stopped_layout(const opb_matcher* m, int32_t* layout) {
  if (!m || !layout || !m->dbg_stopped) return OPB_E_STATE;
  const Layout& L = m->dbg_L;
  const int32_t v[7] = {L.B, L.N, L.M, L.n_pad, L.m_pad, L.R, L.segs()};
  for (int i = 0; i < 7; ++i) layout[i] = v[i];
  return OPB_OK;
}

int opb_debug_read(opb_matcher* m, int32_t which, void* out, size_t capacity_elems, int64_t* n_elems, void* stream) {
  if (!m || !out) return OPB_E_INVALID;
  if (!m->dbg_stopped) return fail(m, OPB_E_STATE, "opb_debug_read: the last forward did not stop (opb_debug_set_stop)");
  cudaStream_t st = (cudaStream_t)stream;
  const Layout& L = m->dbg_L;
  const size_t rows = (size_t)L.rows(), S = (size_t)L.segs();
  const __half *hi = nullptr, *lo = nullptr;    // planes to join, or ...
  const void* raw = nullptr;                    // ... 4- or 8-byte elements to copy
  size_t n = 0, esize = sizeof(float);
  switch (which) {
    case 0: n = rows * kD; hi = m->dbg_x.hi; lo = m->dbg_x.lo; break;
    case 1: n = rows * 512; hi = m->kvt.as<__half>(); break;
    case 2: n = S * kD; raw = m->kmean.p; break;
    case 3: n = S * kD * kD; hi = m->bd.hi.as<__half>(); lo = m->bd.lo.as<__half>(); break;
    case 4: n = rows * kD; hi = m->qp.hi.as<__half>(); lo = m->qp.lo.as<__half>(); break;
    case 5: n = S * 512 * kD; hi = m->g.hi.as<__half>(); lo = m->g.lo.as<__half>(); break;
    case 6: n = rows * 512; raw = m->hid.p; break;
    case 7: n = S * 512; raw = m->mu.p; break;
    case 8: n = S * 512; raw = m->rstd.p; break;
    case 9: n = rows * kD; hi = m->pn.hi.as<__half>(); lo = m->pn.lo.as<__half>(); break;
    case 10: n = (size_t)L.B * L.n_pad; raw = m->rowsum.p; break;
    case 11: n = (size_t)L.B * L.m_pad; raw = m->colsum.p; break;
    case 12: n = (size_t)L.B * L.N; raw = m->rowbest.p; esize = 8; break;
    case 13: n = (size_t)L.B * L.M; raw = m->colbest.p; esize = 8; break;
    case 14:
      if (!m->cfg.with_linear_transform) return fail(m, OPB_E_INVALID, "opb_debug_read: buffer 14 exists with with_linear_transform only");
      n = (size_t)L.B * L.m_pad * kD; hi = m->lin_a.hi.as<__half>(); lo = m->lin_a.lo.as<__half>(); break;
    default: return fail(m, OPB_E_INVALID, "opb_debug_read: unknown buffer %d", which);
  }
  if (n_elems) *n_elems = (int64_t)n;
  if (n > capacity_elems) return fail(m, OPB_E_INVALID, "opb_debug_read: buffer %d has %zu elements, capacity %zu", which, n, capacity_elems);
  if (n == 0) return OPB_OK;
  DeviceGuard dg(m->device);
  CK(m, dg.err);
  return ordered(m, st, [&] {
    if (raw) CK(m, cudaMemcpyAsync(out, raw, n * esize, cudaMemcpyDeviceToDevice, st));
    else join_planes<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(hi, lo, (float*)out, (long long)n);
    CK(m, cudaGetLastError());
    return (int)OPB_OK;
  });
}

int opb_debug_set_ws_fill(int32_t byte) {
  g_ws_fill = byte < 0 ? -1 : (byte & 0xFF);
  return OPB_OK;
}

int opb_debug_set_pdl(int32_t enable) {
  set_pdl_enabled(enable != 0);
  return OPB_OK;
}

int opb_debug_gemm(const opb_debug_gemm_desc* d, void* stream) {
  REQUIRE(__func__, d && d->backend >= 0 && d->backend <= 1 && d->b2_mode >= 0 && d->b2_mode <= 2);
  GemmProblem p{};
  p.epi = d->epi; p.bn = d->bn;
  p.rows = d->rows; p.n_out = d->n_out; p.K1 = d->K1; p.K2 = d->K2;
  p.batch = d->batch ? d->batch : 1;
  p.a_batch_rows = d->a_batch_rows; p.b_batch_rows = d->b_batch_rows;
  p.a1 = CPlanes{(const __half*)d->a1_hi, (const __half*)d->a1_lo, d->a1_ld};
  p.a2 = CPlanes{(const __half*)d->a2_hi, (const __half*)d->a2_lo, d->a2_ld};
  p.b1 = CPlanes{(const __half*)d->b1_hi, (const __half*)d->b1_lo, d->b1_ld};
  p.b2 = CPlanes{(const __half*)d->b2_hi, (const __half*)d->b2_lo, d->b2_ld};
  p.b2_per_seg = d->b2_mode == 1;
  p.b2_lo_zero = d->b2_mode == 2;
  p.a_hi_only = d->a_hi_only;
  p.a_conv = d->a_raw ? 1 : 0; p.a_raw = d->a_raw; p.a_raw_ld = d->a_raw_ld; p.mu = d->mu; p.rstd = d->rstd;
  p.L.B = d->B; p.L.N = d->N; p.L.M = d->M; p.L.n_pad = d->n_pad; p.L.m_pad = d->m_pad; p.L.R = d->n_pad + d->m_pad;
  p.L.nlen = d->nlen; p.L.mlen = d->mlen;
  p.bias = d->bias;
  p.c = d->c; p.ldc = d->ldc; p.c_batch_elems = (long long)d->rows * d->ldc;
  p.out = Planes{(__half*)d->out_hi, (__half*)d->out_lo, d->out_ld};
  p.kmean = d->kmean; p.cross = d->cross; p.statpart = d->statpart;
  p.inv_scale = d->inv_scale; p.rowsum_part = d->rowsum_part; p.colsum_part = d->colsum_part;
  p.inv_rowsum = d->inv_rowsum; p.inv_colsum = d->inv_colsum; p.conf = d->conf; p.conf_ld = d->conf_ld;
  p.rowbest = reinterpret_cast<unsigned long long*>(d->rowbest); p.colbest = reinterpret_cast<unsigned long long*>(d->colbest);
  p.taps = d->taps; p.kb_per_tap = d->kb_per_tap;
  for (int t = 0; t < 9; ++t) p.tap_off[t] = d->tap_off[t];
  p.cv_w2 = d->cv_w2; p.cv_h = d->cv_h; p.cv_w = d->cv_w; p.cv_ppad = d->cv_ppad; p.relu = d->relu; p.range_flag = d->range_flag;
  p.max_ctas = d->max_ctas;
  REQUIRE(__func__, d->backend == 0 || (p.epi == EPI_F32 && !p.a_conv && !p.b2_lo_zero && !p.taps && !p.a_hi_only));   // SIMT: plain product only
  const int rc = d->backend == 1 ? launch_gemm_simt(p, (cudaStream_t)stream) : launch_gemm_tc(p, (cudaStream_t)stream);
  if (rc == 0) return OPB_OK;
  return fail(no_handle_error, rc == -1 ? OPB_E_INVALID : OPB_E_CUDA, "%s: GEMM core of backend %d: %s", __func__, d->backend,
              rc == -1 ? "unsupported problem" : "launch failed");
}

int opb_debug_kv_state_h(const void* kvh, int32_t frames, int32_t n, int32_t m_pts, int32_t slabs_per_group, float* partial, int32_t* n_groups,
                         void* stream) {
  Layout L{};
  L.B = frames; L.N = n; L.M = m_pts; L.n_pad = (n + kSegPad - 1) / kSegPad * kSegPad; L.m_pad = (m_pts + kSegPad - 1) / kSegPad * kSegPad;
  L.R = L.n_pad + L.m_pad;
  int dev = 0, sms = 0;
  CK(no_handle_error, cudaGetDevice(&dev));
  CK(no_handle_error, cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  KvGroups G = kv_groups_for(L, sms);
  if (slabs_per_group > 0) {
    G.slabs = slabs_per_group;
    G.gq = (L.n_pad / 256 + G.slabs - 1) / G.slabs;
    G.gd = (L.m_pad / 256 + G.slabs - 1) / G.slabs;
  }
  if (n_groups) *n_groups = frames * (G.gq + G.gd);
  if (!partial) return OPB_OK;                    // size query
  return launched(__func__, "kv_state_h_kernel", launch_kv_state_h((const __half*)kvh, L, G, partial, (cudaStream_t)stream));
}

int opb_debug_split(const float* x, void* hi, void* lo, size_t n, void* stream) {
  LAUNCH_NH(__func__, split_planes, (unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream, x, (__half*)hi, (__half*)lo, (long long)n);
  return OPB_OK;
}

int opb_debug_block(int32_t prim, int32_t op, int32_t reverse, int32_t threads, int32_t tiles, const void* in, void* value, void* total,
                    void* stream) {
  REQUIRE(__func__, in && value && total);
  REQUIRE(__func__, threads >= 32 && threads <= 1024 && threads % 32 == 0 && tiles > 0);
  REQUIRE(__func__, prim >= 0 && prim <= 2 && op >= 0 && op <= 4);
  REQUIRE(__func__, prim != 2 || op == 0);
  REQUIRE(__func__, reverse == 0 || (prim == 1 && reverse == 1));
  cudaStream_t st = (cudaStream_t)stream;
  const bool rev = reverse != 0;
  if (prim == 2) {
    LAUNCH_NH(__func__, debug_block_rank, 1, threads, 0, st, tiles, (const int32_t*)in, (int32_t*)value, (int32_t*)total);
    return OPB_OK;
  }
  switch (op) {
    case 0: return debug_block_launch<int32_t>(prim, Sum32(), 0, rev, threads, tiles, in, value, total, st);
    case 1: return debug_block_launch<int32_t>(prim, Max(), INT32_MIN, rev, threads, tiles, in, value, total, st);
    case 2: return debug_block_launch<int32_t>(prim, Min(), INT32_MAX, rev, threads, tiles, in, value, total, st);
    case 3: return debug_block_launch<unsigned long long>(prim, Sum64(), 0ull, rev, threads, tiles, in, value, total, st);
    default: return debug_block_launch<long long>(prim, SumS64(), 0ll, rev, threads, tiles, in, value, total, st);
  }
}

}  // extern "C"
