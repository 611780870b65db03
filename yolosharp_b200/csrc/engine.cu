// yolob200 engine: graph construction, weight ingest, workspace planning, forward, C ABI.
//
// The layer list and wiring follow the reference graph definitions
// (Models/Yolo.cs:41-134 Yolov8, :209-257 Yolov11, :337-352 Yolov8Segment) and module
// constructors (Modules/Block.cs, Modules/Head.cs); they are re-expressed as a flat list of
// fused device ops over channel-slice views of NHWC buffers:
//   Conv+BN+SiLU        -> one conv op (BN folded at load, SiLU in the epilogue)
//   chunk / cat         -> producers write channel slices of one wider buffer
//   Bottleneck shortcut -> residual read in the conv epilogue
//   Upsample + Concat   -> copy into the consumer's concat slice
//   SPPF 3x MaxPool     -> one shared-memory kernel writing three slices
//   Detect tail         -> DFL + dist2bbox + sigmoid decode kernel per level
#include <map>
#include <memory>
#include <vector>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <tuple>

#include "common.cuh"

namespace yb {

extern long long* g_tc_dbg;     // conv_tc.cu (debug timeline)
extern int g_tc_dbg_countdown;

static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
bool pdl_enabled() {
  static const bool on = getenv("YB_NO_PDL") == nullptr;
  return on;
}

struct VRef {  // view reference: buffer id + channel slice
  int buf = -1, coff = 0, C = 0;
};

struct BufDesc {
  int H, W, C;
  size_t offset = 0;  // bytes into the arena
};

enum OpType { OP_CONV, OP_DWCONV, OP_POOL, OP_UPSAMPLE, OP_DECODE, OP_PROTO_OUT, OP_PIXSHUF, OP_ATTN };

struct OpDesc {
  OpType type;
  std::string name;  // reference module path ("model.2.m.0.cv1") or a descriptive tag
  VRef in, out, res, out2, out3;
  int k = 1, s = 1, act = ACT_SILU, cin = 0, cout = 0, groups = 1;
  bool bn = true;        // Conv (conv+bn) vs plain Conv2d(bias)
  bool convt = false;    // weights come from a ConvTranspose2d(c,c,2,2) [Cin][Cout][2][2]: run as 1x1 conv to 4*c
  int nh = 0, kd = 0, hd = 0;  // attention
  float scale = 0.f;
  // decode
  int level = 0, a0 = 0;
  float stride = 0;
  VRef cls, coef;
  // device weights
  float* w_f32 = nullptr;   // generic layout [tap][Cin][Cout] (or [9][C] depthwise)
  __half* w_f16 = nullptr;  // tensor-core layout [Cout][tap*Cin]
  float* bias = nullptr;
  TcConvPlan* plan = nullptr;
  bool use_tc = false;
  std::vector<std::string> parts;  // merged conv: reference names whose output channels are concatenated
  std::vector<int> part_cout;
  int fork_id = -1;    // after this op: record ev_fork[fork_id] (sibling lanes wait for it)
  int wait_fork = -1;  // lane start waits for ev_fork[wait_fork] instead of the level's feature event
  int lane = 0;        // 0 = main stream; >0 = independent head branch that may run concurrently
  int lane_level = -1; // pyramid level whose feature map a side lane waits for
  int feat_level = -1; // this op completes feats[feat_level] (fork point for the head lanes)
  EpiDecode dec;       // conv: fused Detect-tail epilogue (tensor-core path)
  bool fused = false;  // decode op: its work is done by the producing convs' epilogues
  TcBneckPlan* bneck = nullptr;  // conv: fused Bottleneck that also computes the previous op (its input) in smem
  bool absorbed = false;         // conv: computed inside the next op's fused launch (Bottleneck or fold); launches nothing
  TcConvPlan* fold = nullptr;    // 1x1 conv: plan that also computes the previous op, its input never leaving registers
  bool folded = false;           // conv: absorbed into the next op's fold
};

struct HostTensor {
  std::vector<float> data;
  std::vector<int64_t> shape;
};

}  // namespace yb

using namespace yb;

struct yb_engine {
  yb_config cfg;
  std::vector<BufDesc> bufs;
  std::vector<OpDesc> ops;
  std::map<std::string, HostTensor> host;
  std::vector<std::string> expected;
  char* arena = nullptr;
  size_t arena_bytes = 0;
  int* tile_ctr = nullptr;  // one dynamic-scheduler counter per op, zeroed at the start of every forward
  int src_h = 0, src_w = 0;  // size of the caller's (unpadded) images for the forward being enqueued (yb_forward_padded)
  bool finalized = false;
  int esize = 4;  // bytes per activation element
  int A = 0, pred_c = 0;
  int widths[5];
  int ch[3];
  VRef input_nhwc;  // generic path: converted network input (3 channels)
  VRef proto_view;
  bool has_stem_tc = false;
  // staging for yb_predict_u8 (index 0) and the pipelined slots of yb_predict_u8_submit (1 .. kSlots)
  struct Stage {
    uint8_t* in = nullptr;
    float* pred = nullptr;
    float* dets = nullptr;
    int* counts = nullptr;
    int max_det = 0;
    float* proto = nullptr;    // segment engines
    uint8_t* masks = nullptr;  // (max_batch, mask_cap, H, W)
    int mask_cap = 0;
    cudaStream_t stream = nullptr;
  };
  static const int kSlots = 4;
  Stage stage[1 + kSlots];
  cudaEvent_t arena_free = nullptr;  // recorded after each staged forward: the activation arena is shared
  bool arena_used = false;
  // CUDA graph cache
  struct GraphKey {
    const void* in; int dtype; int B; float* pred; float* proto; int src_h, src_w;
    bool operator<(const GraphKey& o) const {
      return std::tie(in, dtype, B, pred, proto, src_h, src_w) < std::tie(o.in, o.dtype, o.B, o.pred, o.proto, o.src_h, o.src_w);
    }
  };
  std::map<GraphKey, cudaGraphExec_t> graphs;
  std::map<GraphKey, int> seen;
  cudaStream_t capture_stream = nullptr;
  std::vector<void*> dev_allocs;
  // concurrent head branches (box / cls / mask-coefficient chains of the three levels + Proto)
  static const int kLanes = 13;
  cudaStream_t side[kLanes] = {};
  cudaEvent_t ev_feat[3] = {}, ev_done[kLanes] = {}, ev_fork[3] = {};
  bool lanes_ok = false;
};

namespace yb {

// ------------------------------------------------------------------------------------------
// Graph builder
// ------------------------------------------------------------------------------------------
struct Builder {
  yb_engine* e;
  VRef new_buf(int H, int W, int C) {
    e->bufs.push_back({H, W, C, 0});
    return VRef{(int)e->bufs.size() - 1, 0, C};
  }
  static VRef slice(VRef v, int coff, int C) { return VRef{v.buf, v.coff + coff, C}; }
  int H(VRef v) const { return e->bufs[v.buf].H; }
  int W(VRef v) const { return e->bufs[v.buf].W; }

  // Convs.Conv (Modules/Convs.cs:36-56) or plain Conv2d(bias) when bn == false
  void conv(const std::string& name, VRef in, VRef out, int k, int s, int act = ACT_SILU, bool bn = true,
            VRef res = VRef(), int groups = 1) {
    OpDesc op;
    op.type = groups == 1 ? OP_CONV : OP_DWCONV;
    op.name = name;
    op.in = in; op.out = out; op.res = res;
    op.k = k; op.s = s; op.act = act; op.cin = in.C; op.cout = out.C; op.bn = bn; op.groups = groups;
    e->ops.push_back(op);
    if (bn) {
      for (const char* sfx : {".conv.weight", ".bn.weight", ".bn.bias", ".bn.running_mean", ".bn.running_var"})
        e->expected.push_back(name + sfx);
    } else {
      e->expected.push_back(name + ".weight");
      e->expected.push_back(name + ".bias");
    }
  }

  // Several Conv modules that read the SAME input (the first convs of the Detect branches, Head.cs:47-49)
  // as one conv whose output channels are the concatenation of theirs: one pass over the input and a
  // wider N per wgmma (N = 144 instead of 64 and 80).
  void conv_merged(const std::vector<std::string>& names, const std::vector<int>& couts, VRef in, VRef out, int k, int s) {
    OpDesc op;
    op.type = OP_CONV;
    op.name = names[0];
    for (size_t i = 1; i < names.size(); i++) op.name += "+" + names[i].substr(names[i].rfind(".cv") + 1);
    op.in = in; op.out = out;
    op.k = k; op.s = s; op.act = ACT_SILU; op.cin = in.C; op.cout = out.C; op.bn = true;
    op.parts = names; op.part_cout = couts;
    e->ops.push_back(op);
    for (const auto& n : names)
      for (const char* sfx : {".conv.weight", ".bn.weight", ".bn.bias", ".bn.running_mean", ".bn.running_var"})
        e->expected.push_back(n + sfx);
  }

  // Block.Bottleneck (Block.cs:572-607)
  void bottleneck(const std::string& name, VRef in, VRef out, bool shortcut, int k0, int k1, double ex) {
    const int c_ = (int)(out.C * ex);
    VRef t = new_buf(H(in), W(in), c_);
    conv(name + ".cv1", in, t, k0, 1);
    conv(name + ".cv2", t, out, k1, 1, ACT_SILU, true, (shortcut && in.C == out.C) ? in : VRef());
  }

  // Block.C2f (Block.cs:371-398): cv1 -> 2 chunks; each Bottleneck(c,c,e=1.0) appends a slice; cv2 on the cat
  void c2f(const std::string& name, VRef in, VRef out, int n, bool shortcut) {
    const int c = (int)(out.C * 0.5);
    VRef cat = new_buf(H(in), W(in), (2 + n) * c);
    conv(name + ".cv1", in, slice(cat, 0, 2 * c), 1, 1);
    for (int i = 0; i < n; i++)
      bottleneck(name + ".m." + std::to_string(i), slice(cat, (1 + i) * c, c), slice(cat, (2 + i) * c, c), shortcut,
                 3, 3, 1.0);
    conv(name + ".cv2", cat, out, 1, 1);
  }

  // Block.C3k (Block.cs:611-620 over C3 :404-441): cv3(cat(m(cv1 x), cv2 x)), m = n x Bottleneck(k 3,3 e 1.0)
  void c3k(const std::string& name, VRef in, VRef out, int n, bool shortcut) {
    const int c_ = (int)(out.C * 0.5);
    VRef cat = new_buf(H(in), W(in), 2 * c_);
    VRef cur = new_buf(H(in), W(in), c_);
    conv(name + ".cv1", in, cur, 1, 1);
    for (int i = 0; i < n; i++) {
      VRef nxt = (i == n - 1) ? slice(cat, 0, c_) : new_buf(H(in), W(in), c_);
      bottleneck(name + ".m." + std::to_string(i), cur, nxt, shortcut, 3, 3, 1.0);
      cur = nxt;
    }
    conv(name + ".cv2", in, slice(cat, c_, c_), 1, 1);
    conv(name + ".cv3", cat, out, 1, 1);
  }

  // Block.C3k2 (Block.cs:623-661)
  void c3k2(const std::string& name, VRef in, VRef out, int n, bool use_c3k, double ex, bool shortcut = true) {
    const int c = (int)(out.C * ex);
    VRef cat = new_buf(H(in), W(in), (2 + n) * c);
    conv(name + ".cv1", in, slice(cat, 0, 2 * c), 1, 1);
    for (int i = 0; i < n; i++) {
      VRef bi = slice(cat, (1 + i) * c, c), bo = slice(cat, (2 + i) * c, c);
      if (use_c3k) c3k(name + ".m." + std::to_string(i), bi, bo, 2, shortcut);
      else bottleneck(name + ".m." + std::to_string(i), bi, bo, shortcut, 3, 3, 0.5);
    }
    conv(name + ".cv2", cat, out, 1, 1);
  }

  // Block.SPPF (Block.cs:236-282): cv1 has no activation (reference quirk, :257)
  void sppf(const std::string& name, VRef in, VRef out) {
    const int c_ = in.C / 2;
    VRef cat = new_buf(H(in), W(in), 4 * c_);
    conv(name + ".cv1", in, slice(cat, 0, c_), 1, 1, ACT_NONE);
    OpDesc op;
    op.type = OP_POOL;
    op.name = name + ".m";
    op.in = slice(cat, 0, c_);
    op.out = slice(cat, c_, c_);
    op.out2 = slice(cat, 2 * c_, c_);
    op.out3 = slice(cat, 3 * c_, c_);
    e->ops.push_back(op);
    conv(name + ".cv2", cat, out, 1, 1);
  }

  // Convs.DWConv (Convs.cs:108-114): groups = gcd(c1,c2) = c for the square cases used by v11
  void dwconv(const std::string& name, VRef in, VRef out, VRef res = VRef()) {
    conv(name, in, out, 3, 1, ACT_SILU, true, res, in.C);
  }

  // Block.Attention + PSABlock + C2PSA (Block.cs:664-810).  All convs keep SiLU (reference quirk).
  void c2psa(const std::string& name, VRef in, VRef out, int n) {
    const int c = (int)(in.C * 0.5);
    const int h = H(in), w = W(in);
    VRef cat = new_buf(h, w, 2 * c);
    conv(name + ".cv1", in, cat, 1, 1);
    VRef b = slice(cat, c, c);
    const int nh = c / 64, hd = c / nh, kd = (int)(hd * 0.5);
    for (int i = 0; i < n; i++) {
      const std::string bn = name + ".m." + std::to_string(i);
      VRef qkv = new_buf(h, w, c + 2 * nh * kd);
      conv(bn + ".attn.qkv", b, qkv, 1, 1);
      VRef ao = new_buf(h, w, c), vd = new_buf(h, w, c), xs = new_buf(h, w, c), b1 = new_buf(h, w, c);
      OpDesc op;
      op.type = OP_ATTN;
      op.name = bn + ".attn.core";
      op.in = qkv; op.out = ao; op.out2 = vd;
      op.nh = nh; op.kd = kd; op.hd = hd;
      op.scale = (float)std::pow((double)kd, -0.5);
      e->ops.push_back(op);
      dwconv(bn + ".attn.pe", vd, xs, ao);           // attn_out + pe(v)
      conv(bn + ".attn.proj", xs, b1, 1, 1, ACT_SILU, true, b);  // b + attn(b)
      VRef f = new_buf(h, w, 2 * c);
      conv(bn + ".ffn.0", b1, f, 1, 1);
      conv(bn + ".ffn.1", f, b, 1, 1, ACT_SILU, true, b1);      // b1 + ffn(b1), back into the cat slice
    }
    conv(name + ".cv2", cat, out, 1, 1);
  }

  // Block.Proto (Block.cs:51-84): Conv3x3 -> ConvTranspose2d(2,2) -> Conv3x3 -> Conv1x1
  VRef proto(const std::string& name, VRef in, int npr, int nm) {
    const int h = H(in), w = W(in);
    VRef p1 = new_buf(h, w, npr);
    conv(name + ".cv1", in, p1, 3, 1);
    VRef up4 = new_buf(h, w, 4 * npr);
    conv(name + ".upsample", p1, up4, 1, 1, ACT_NONE, false);
    e->ops.back().convt = true;
    VRef up = new_buf(2 * h, 2 * w, npr);
    OpDesc op;
    op.type = OP_PIXSHUF;
    op.name = name + ".upsample.shuffle";
    op.in = up4; op.out = up;
    e->ops.push_back(op);
    VRef p2 = new_buf(2 * h, 2 * w, npr);
    conv(name + ".cv2", up, p2, 3, 1);
    VRef p3 = new_buf(2 * h, 2 * w, nm);
    conv(name + ".cv3", p2, p3, 1, 1);
    OpDesc po;
    po.type = OP_PROTO_OUT;
    po.name = name + ".out";
    po.in = p3; po.out = p3;
    e->ops.push_back(po);
    return p3;
  }

  void upsample(const std::string& name, VRef in, VRef out) {
    OpDesc op;
    op.type = OP_UPSAMPLE;
    op.name = name;
    op.in = in; op.out = out;
    e->ops.push_back(op);
  }
};

static int build_graph(yb_engine* e) {
  const yb_config& c = e->cfg;
  Builder b{e};
  const int H = c.height, W = c.width;
  int w[5];
  int n3[3];  // C2f depths
  bool v11 = c.arch == YB_ARCH_V11;
  bool use_c3k = false;
  int n11 = 1;
  if (!v11) {
    // Yolo.cs:45-49
    static const float dm[5] = {0.34f, 0.34f, 0.67f, 1.0f, 1.0f};
    static const float wm[5] = {0.25f, 0.5f, 0.75f, 1.0f, 1.25f};
    static const int mc[5] = {1024, 1024, 576, 512, 640};
    const int base[5] = {64, 128, 256, 512, 1024};
    for (int i = 0; i < 5; i++) w[i] = std::min((int)(base[i] * wm[c.size]), mc[c.size]);
    const int d[3] = {3, 6, 9};
    for (int i = 0; i < 3; i++) n3[i] = (int)(d[i] * dm[c.size]);
  } else {
    // Yolo.cs:213-217
    static const float dm[5] = {0.5f, 0.5f, 0.5f, 1.0f, 1.0f};
    static const float wm[5] = {0.25f, 0.5f, 1.0f, 1.0f, 1.5f};
    static const int mc[5] = {1024, 1024, 512, 512, 768};
    static const bool ck[5] = {false, false, true, true, true};
    const int base[5] = {64, 128, 256, 512, 1024};
    for (int i = 0; i < 5; i++) w[i] = std::min((int)(base[i] * wm[c.size]), mc[c.size]);
    n11 = (int)(2 * dm[c.size]);
    use_c3k = ck[c.size];
  }
  for (int i = 0; i < 5; i++) e->widths[i] = w[i];
  e->ch[0] = w[2]; e->ch[1] = w[3]; e->ch[2] = w[4];

  // generic path reads the network input through an NHWC copy (3 channels)
  e->input_nhwc = b.new_buf(H, W, 3);
  auto M = [](int i) { return "model." + std::to_string(i); };

  VRef p3, p4, p5;  // Detect inputs
  if (!v11) {
    // concat buffers (Yolo.cs:70-84; Concat order = [x, saved])
    VRef cat11 = b.new_buf(H / 16, W / 16, w[4] + w[3]);  // [up(L9), L6]
    VRef cat14 = b.new_buf(H / 8, W / 8, w[3] + w[2]);    // [up(L12), L4]
    VRef cat17 = b.new_buf(H / 16, W / 16, w[2] + w[3]);  // [L16, L12]
    VRef cat20 = b.new_buf(H / 32, W / 32, w[3] + w[4]);  // [L19, L9]
    VRef l0 = b.new_buf(H / 2, W / 2, w[0]);
    b.conv(M(0), e->input_nhwc, l0, 3, 2);
    VRef l1 = b.new_buf(H / 4, W / 4, w[1]);
    b.conv(M(1), l0, l1, 3, 2);
    VRef l2 = b.new_buf(H / 4, W / 4, w[1]);
    b.c2f(M(2), l1, l2, n3[0], true);
    VRef l3 = b.new_buf(H / 8, W / 8, w[2]);
    b.conv(M(3), l2, l3, 3, 2);
    VRef l4 = Builder::slice(cat14, w[3], w[2]);
    b.c2f(M(4), l3, l4, n3[1], true);
    VRef l5 = b.new_buf(H / 16, W / 16, w[3]);
    b.conv(M(5), l4, l5, 3, 2);
    VRef l6 = Builder::slice(cat11, w[4], w[3]);
    b.c2f(M(6), l5, l6, n3[1], true);
    VRef l7 = b.new_buf(H / 32, W / 32, w[4]);
    b.conv(M(7), l6, l7, 3, 2);
    VRef l8 = b.new_buf(H / 32, W / 32, w[4]);
    b.c2f(M(8), l7, l8, n3[0], true);
    VRef l9 = Builder::slice(cat20, w[3], w[4]);
    b.sppf(M(9), l8, l9);
    b.upsample(M(10), l9, Builder::slice(cat11, 0, w[4]));
    VRef l12 = Builder::slice(cat17, w[2], w[3]);
    b.c2f(M(12), cat11, l12, n3[0], false);
    b.upsample(M(13), l12, Builder::slice(cat14, 0, w[3]));
    VRef l15 = b.new_buf(H / 8, W / 8, w[2]);
    b.c2f(M(15), cat14, l15, n3[0], false);
    b.conv(M(16), l15, Builder::slice(cat17, 0, w[2]), 3, 2);
    VRef l18 = b.new_buf(H / 16, W / 16, w[3]);
    b.c2f(M(18), cat17, l18, n3[0], false);
    b.conv(M(19), l18, Builder::slice(cat20, 0, w[3]), 3, 2);
    VRef l21 = b.new_buf(H / 32, W / 32, w[4]);
    b.c2f(M(21), cat20, l21, n3[0], false);
    p3 = l15; p4 = l18; p5 = l21;
  } else {
    // Yolo.cs:209-257; saved outputs {4,6,10,13,16,19,22}, concat partners {6,4,13,10}
    VRef cat12 = b.new_buf(H / 16, W / 16, w[4] + w[3]);  // [up(L10), L6]
    VRef cat15 = b.new_buf(H / 8, W / 8, w[3] + w[3]);    // [up(L13), L4]
    VRef cat18 = b.new_buf(H / 16, W / 16, w[2] + w[3]);  // [L17, L13]
    VRef cat21 = b.new_buf(H / 32, W / 32, w[3] + w[4]);  // [L20, L10]
    VRef l0 = b.new_buf(H / 2, W / 2, w[0]);
    b.conv(M(0), e->input_nhwc, l0, 3, 2);
    VRef l1 = b.new_buf(H / 4, W / 4, w[1]);
    b.conv(M(1), l0, l1, 3, 2);
    VRef l2 = b.new_buf(H / 4, W / 4, w[2]);
    b.c3k2(M(2), l1, l2, n11, use_c3k, 0.25);
    VRef l3 = b.new_buf(H / 8, W / 8, w[2]);
    b.conv(M(3), l2, l3, 3, 2);
    VRef l4 = Builder::slice(cat15, w[3], w[3]);
    b.c3k2(M(4), l3, l4, n11, use_c3k, 0.25);
    VRef l5 = b.new_buf(H / 16, W / 16, w[3]);
    b.conv(M(5), l4, l5, 3, 2);
    VRef l6 = Builder::slice(cat12, w[4], w[3]);
    b.c3k2(M(6), l5, l6, n11, true, 0.5);
    VRef l7 = b.new_buf(H / 32, W / 32, w[4]);
    b.conv(M(7), l6, l7, 3, 2);
    VRef l8 = b.new_buf(H / 32, W / 32, w[4]);
    b.c3k2(M(8), l7, l8, n11, true, 0.5);
    VRef l9 = b.new_buf(H / 32, W / 32, w[4]);
    b.sppf(M(9), l8, l9);
    VRef l10 = Builder::slice(cat21, w[3], w[4]);
    b.c2psa(M(10), l9, l10, n11);
    b.upsample(M(11), l10, Builder::slice(cat12, 0, w[4]));
    VRef l13 = Builder::slice(cat18, w[2], w[3]);
    b.c3k2(M(13), cat12, l13, n11, use_c3k, 0.5);
    b.upsample(M(14), l13, Builder::slice(cat15, 0, w[3]));
    VRef l16 = b.new_buf(H / 8, W / 8, w[2]);
    b.c3k2(M(16), cat15, l16, n11, use_c3k, 0.5);
    b.conv(M(17), l16, Builder::slice(cat18, 0, w[2]), 3, 2);
    VRef l19 = b.new_buf(H / 16, W / 16, w[3]);
    b.c3k2(M(19), cat18, l19, n11, use_c3k, 0.5);
    b.conv(M(20), l19, Builder::slice(cat21, 0, w[3]), 3, 2);
    VRef l22 = b.new_buf(H / 32, W / 32, w[4]);
    b.c3k2(M(22), cat21, l22, n11, true, 0.5);
    p3 = l16; p4 = l19; p5 = l22;
  }

  // ---- Detect / Segment head (Head.cs:35-53, 247-259) ----
  const int head = v11 ? 23 : 22;
  const std::string hn = M(head);
  const int nc = c.nc, rm = c.reg_max;
  const int c2 = std::max(16, std::max(e->ch[0] / 4, rm * 4));
  const int c3 = std::max(e->ch[0], std::min(nc, 100));
  const bool seg = c.task == YB_TASK_SEGMENT;
  const int nm = 32;
  const int c4 = std::max(e->ch[0] / 4, nm);
  VRef feats[3] = {p3, p4, p5};
  const int strides[3] = {8, 16, 32};
  e->A = 0;
  for (int l = 0; l < 3; l++) e->A += (H / strides[l]) * (W / strides[l]);
  e->pred_c = 4 + nc + (seg ? nm : 0);
  int a0 = 0;
  for (int l = 0; l < 3; l++)  // fork points: the last op that writes each Detect input
    for (int i = (int)e->ops.size() - 1; i >= 0; i--)
      if (e->ops[i].out.buf == feats[l].buf) { e->ops[i].feat_level = l; break; }
  auto tag_lane = [&](size_t from, int lane, int level) {
    for (size_t i = from; i < e->ops.size(); i++) { e->ops[i].lane = lane; e->ops[i].lane_level = level; }
  };
  for (int l = 0; l < 3; l++) {
    const int hl = H / strides[l], wl = W / strides[l];
    const std::string L = std::to_string(l);
    size_t mark = e->ops.size();
    const bool merge = !v11;  // legacy head: cv2[l][0], cv3[l][0] (and cv4[l][0]) are 3x3 Convs of the same input
    VRef t1, u1, m1;
    if (merge) {
      std::vector<std::string> names = {hn + ".cv2." + L + ".0", hn + ".cv3." + L + ".0"};
      std::vector<int> couts = {c2, c3};
      if (seg) { names.push_back(hn + ".cv4." + L + ".0"); couts.push_back(c4); }
      VRef first = b.new_buf(hl, wl, c2 + c3 + (seg ? c4 : 0));
      b.conv_merged(names, couts, feats[l], first, 3, 1);
      e->ops.back().fork_id = l;
      t1 = Builder::slice(first, 0, c2);
      u1 = Builder::slice(first, c2, c3);
      if (seg) m1 = Builder::slice(first, c2 + c3, c4);
    } else {
      t1 = b.new_buf(hl, wl, c2);
      b.conv(hn + ".cv2." + L + ".0", feats[l], t1, 3, 1);
    }
    VRef t2 = b.new_buf(hl, wl, c2), box = b.new_buf(hl, wl, 4 * rm);
    b.conv(hn + ".cv2." + L + ".1", t1, t2, 3, 1);
    b.conv(hn + ".cv2." + L + ".2", t2, box, 1, 1, ACT_NONE, false);
    tag_lane(mark, 1 + 3 * l, l);
    mark = e->ops.size();
    VRef u2 = b.new_buf(hl, wl, c3), cls = b.new_buf(hl, wl, nc);
    if (!v11) {  // legacy cls branch: two 3x3 Convs (Head.cs:49); the first one is part of the merged conv
      b.conv(hn + ".cv3." + L + ".1", u1, u2, 3, 1);
    } else {     // Head.cs:50: [DW3x3(x) + Conv1x1(x->c3)] . [DW3x3(c3) + Conv1x1(c3->c3)]
      u1 = b.new_buf(hl, wl, c3);
      VRef d1 = b.new_buf(hl, wl, feats[l].C), d2 = b.new_buf(hl, wl, c3);
      b.dwconv(hn + ".cv3." + L + ".0.0", feats[l], d1);
      b.conv(hn + ".cv3." + L + ".0.1", d1, u1, 1, 1);
      b.dwconv(hn + ".cv3." + L + ".1.0", u1, d2);
      b.conv(hn + ".cv3." + L + ".1.1", d2, u2, 1, 1);
    }
    b.conv(hn + ".cv3." + L + ".2", u2, cls, 1, 1, ACT_NONE, false);
    tag_lane(mark, 2 + 3 * l, l);
    if (merge) for (size_t i = mark; i < e->ops.size(); i++) e->ops[i].wait_fork = l;
    mark = e->ops.size();
    VRef coef;
    if (seg) {
      VRef m2 = b.new_buf(hl, wl, c4);
      coef = b.new_buf(hl, wl, nm);
      if (!merge) {
        m1 = b.new_buf(hl, wl, c4);
        b.conv(hn + ".cv4." + L + ".0", feats[l], m1, 3, 1);
      }
      b.conv(hn + ".cv4." + L + ".1", m1, m2, 3, 1);
      b.conv(hn + ".cv4." + L + ".2", m2, coef, 1, 1, ACT_NONE, false);
      tag_lane(mark, 3 + 3 * l, l);
      if (merge) for (size_t i = mark; i < e->ops.size(); i++) e->ops[i].wait_fork = l;
    }
    OpDesc op;
    op.type = OP_DECODE;
    op.name = hn + ".decode." + L;
    op.in = box; op.cls = cls; op.coef = coef;
    op.level = l; op.a0 = a0; op.stride = (float)strides[l];
    e->ops.push_back(op);
    a0 += hl * wl;
  }
  if (seg) {
    const size_t mark = e->ops.size();
    e->proto_view = b.proto(hn + ".proto", feats[0], e->ch[0], nm);  // Head.cs:247: npr = ch[0]
    tag_lane(mark, 10, 0);
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// Weights
// ------------------------------------------------------------------------------------------
static const HostTensor* find_tensor(yb_engine* e, const std::string& name) {
  auto it = e->host.find(name);
  if (it == e->host.end()) {
    set_error("missing weight tensor: " + name);
    return nullptr;
  }
  return &it->second;
}

static float round_f16(float v) { return __half2float(__float2half_rn(v)); }

template <typename T>
static int upload(yb_engine* e, const std::vector<T>& h, T** dptr) {
  YB_CUDA_CHECK(cudaMalloc((void**)dptr, h.size() * sizeof(T)));
  e->dev_allocs.push_back(*dptr);
  YB_CUDA_CHECK(cudaMemcpy(*dptr, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  return 0;
}

static int finalize_conv(yb_engine* e, OpDesc& op) {
  if (!op.parts.empty() && e->host.find(op.name + ".conv.weight") == e->host.end()) {
    // merged conv: synthesise concatenated tensors under the merged name, then fold as usual
    HostTensor W, g, bt, mu, var;
    for (const auto& n : op.parts) {
      const HostTensor *w1 = find_tensor(e, n + ".conv.weight"), *g1 = find_tensor(e, n + ".bn.weight"),
                       *b1 = find_tensor(e, n + ".bn.bias"), *m1 = find_tensor(e, n + ".bn.running_mean"),
                       *v1 = find_tensor(e, n + ".bn.running_var");
      if (!w1 || !g1 || !b1 || !m1 || !v1) return YB_ERR_MISSING_WEIGHT;
      W.data.insert(W.data.end(), w1->data.begin(), w1->data.end());
      g.data.insert(g.data.end(), g1->data.begin(), g1->data.end());
      bt.data.insert(bt.data.end(), b1->data.begin(), b1->data.end());
      mu.data.insert(mu.data.end(), m1->data.begin(), m1->data.end());
      var.data.insert(var.data.end(), v1->data.begin(), v1->data.end());
    }
    e->host[op.name + ".conv.weight"] = W;
    e->host[op.name + ".bn.weight"] = g;
    e->host[op.name + ".bn.bias"] = bt;
    e->host[op.name + ".bn.running_mean"] = mu;
    e->host[op.name + ".bn.running_var"] = var;
  }
  const bool f16 = e->cfg.precision == YB_PREC_F16;
  const int taps = op.k * op.k;
  const int cing = op.cin / op.groups;  // input channels per group
  const HostTensor* W = find_tensor(e, op.name + (op.bn ? ".conv.weight" : ".weight"));
  if (!W) return YB_ERR_MISSING_WEIGHT;
  if ((int64_t)W->data.size() != (int64_t)op.cout * cing * taps) {
    set_error("shape mismatch for " + op.name + " weight");
    return YB_ERR_SHAPE;
  }
  HostTensor Wt;  // ConvTranspose2d [Cin][Cout][2][2] -> 1x1 conv weight [(i*2+j)*Cout + co][Cin]
  if (op.convt) {
    const int cr = op.cout / 4;
    Wt.data.resize(W->data.size());
    for (int ci = 0; ci < op.cin; ci++)
      for (int co = 0; co < cr; co++)
        for (int ph = 0; ph < 4; ph++) Wt.data[((size_t)ph * cr + co) * op.cin + ci] = W->data[((size_t)ci * cr + co) * 4 + ph];
    W = &Wt;
  }
  std::vector<double> scale(op.cout, 1.0);
  std::vector<float> bias(op.cout, 0.f);
  if (op.bn) {
    const HostTensor *g = find_tensor(e, op.name + ".bn.weight"), *bt = find_tensor(e, op.name + ".bn.bias"),
                     *mu = find_tensor(e, op.name + ".bn.running_mean"),
                     *var = find_tensor(e, op.name + ".bn.running_var");
    if (!g || !bt || !mu || !var) return YB_ERR_MISSING_WEIGHT;
    if ((int)g->data.size() != op.cout || (int)bt->data.size() != op.cout || (int)mu->data.size() != op.cout ||
        (int)var->data.size() != op.cout) {
      set_error("shape mismatch for " + op.name + " bn");
      return YB_ERR_SHAPE;
    }
    for (int o = 0; o < op.cout; o++) {
      // eval-mode BatchNorm2d, eps = 1e-3 (Modules/Convs.cs:41)
      scale[o] = (double)g->data[o] / std::sqrt((double)var->data[o] + 1e-3);
      bias[o] = (float)((double)bt->data[o] - (double)mu->data[o] * scale[o]);
    }
  } else {
    const HostTensor* bb = find_tensor(e, op.name + ".bias");
    if (!bb) return YB_ERR_MISSING_WEIGHT;
    const int breal = op.convt ? op.cout / 4 : op.cout;
    if ((int)bb->data.size() != breal) {
      set_error("shape mismatch for " + op.name + " bias");
      return YB_ERR_SHAPE;
    }
    for (int o = 0; o < op.cout; o++) bias[o] = bb->data[o % breal];
  }
  // folded weight (o, ci, kh, kw) -> fp32; in F16 mode rounded through fp16 so that the CUDA-core
  // twin and the tensor-core kernel see identical operand values
  std::vector<float> wf((size_t)op.cout * cing * taps);
  for (int o = 0; o < op.cout; o++)
    for (int ci = 0; ci < cing; ci++)
      for (int t = 0; t < taps; t++) {
        float v = (float)((double)W->data[((size_t)o * cing + ci) * taps + t] * scale[o]);
        if (f16) v = round_f16(v);
        wf[((size_t)o * cing + ci) * taps + t] = v;
      }
  if (upload(e, bias, &op.bias)) return YB_ERR_CUDA;
  if (op.type == OP_DWCONV) {
    if (op.groups != op.cin || op.cin != op.cout || op.k != 3 || op.s != 1) {
      set_error("only depthwise 3x3 s1 grouped convs are supported: " + op.name);
      return YB_ERR_NOT_IMPLEMENTED;
    }
    std::vector<float> g9((size_t)9 * op.cout);
    for (int o = 0; o < op.cout; o++)
      for (int t = 0; t < 9; t++) g9[(size_t)t * op.cout + o] = wf[(size_t)o * 9 + t];
    return upload(e, g9, &op.w_f32);
  }
  // generic layout [tap][Cin][Cout]
  std::vector<float> wg((size_t)taps * op.cin * op.cout);
  for (int o = 0; o < op.cout; o++)
    for (int ci = 0; ci < op.cin; ci++)
      for (int t = 0; t < taps; t++)
        wg[((size_t)t * op.cin + ci) * op.cout + o] = wf[((size_t)o * op.cin + ci) * taps + t];
  if (upload(e, wg, &op.w_f32)) return YB_ERR_CUDA;
  if (f16) {
    // tensor-core layout [Cout][tap][Cin] (K-major rows for the wgmma B operand)
    std::vector<__half> wh((size_t)op.cout * taps * op.cin);
    for (int o = 0; o < op.cout; o++)
      for (int t = 0; t < taps; t++)
        for (int ci = 0; ci < op.cin; ci++)
          wh[((size_t)o * taps + t) * op.cin + ci] = __float2half_rn(wf[((size_t)o * op.cin + ci) * taps + t]);
    if (op.cin == 3 && op.k == 3) {
      // stem: k = (kh*3 + c)*4 + kw + 1, K = 36 padded to 64 (see stem_tc_kernel)
      wh.assign((size_t)op.cout * 64, __float2half_rn(0.f));
      for (int o = 0; o < op.cout; o++)
        for (int kh = 0; kh < 3; kh++)
          for (int ci = 0; ci < 3; ci++)
            for (int kw = 0; kw < 3; kw++)
              wh[(size_t)o * 64 + (kh * 3 + ci) * 4 + kw + 1] = __float2half_rn(wf[((size_t)o * 3 + ci) * 9 + kh * 3 + kw]);
    }
    if (upload(e, wh, &op.w_f16)) return YB_ERR_CUDA;
  }
  return 0;
}

static View make_view(const yb_engine* e, VRef r) {
  View v;
  if (r.buf < 0) return v;
  const BufDesc& b = e->bufs[r.buf];
  v.base = e->arena + b.offset;
  v.H = b.H; v.W = b.W; v.pitch = b.C; v.coff = r.coff; v.C = r.C;
  return v;
}

static ConvParams conv_params(const yb_engine* e, const OpDesc& op, int B) {
  ConvParams p;
  p.in = make_view(e, op.in);
  p.out = make_view(e, op.out);
  p.res = make_view(e, op.res);
  p.w = op.w_f32;
  p.bias = op.bias;
  p.B = B;
  p.Cin = op.cin; p.Cout = op.cout;
  p.k = op.k; p.stride = op.s; p.pad = op.k / 2;
  p.Ho = p.out.H; p.Wo = p.out.W;
  p.act = op.act;
  return p;
}

template <typename T>
static int run_ops(yb_engine* e, const void* in, int in_dtype, int B, float* out_pred, float* out_proto,
                   cudaStream_t s, cudaEvent_t* events = nullptr, int only = -1) {
  int rc;
  bool input_converted = false;
  // Head branches are independent chains of small, latency-bound kernels: with every Detect tail fused
  // (tensor-core path) they run on side streams forked at the op that completes their feature map and are
  // joined at the end; inside a captured CUDA graph this becomes real branch parallelism.
  const bool lanes = e->lanes_ok && !events && only < 0;
  bool lane_started[yb_engine::kLanes] = {};
  cudaStream_t main_s = s;
  if (only >= 0) input_converted = true;  // single-op timing (yb_time_op): buffers hold the last forward's data
  if (e->tile_ctr)
    YB_CUDA_CHECK(cudaMemsetAsync(e->tile_ctr, 0, e->ops.size() * sizeof(int), s));
  for (size_t i = 0; i < e->ops.size(); i++) {
    if (only >= 0 && (int)i != only) continue;
    OpDesc& op = e->ops[i];
    s = main_s;
    if (lanes && op.lane > 0) {
      s = e->side[op.lane];
      if (!lane_started[op.lane]) {
        YB_CUDA_CHECK(cudaStreamWaitEvent(s, op.wait_fork >= 0 ? e->ev_fork[op.wait_fork] : e->ev_feat[op.lane_level], 0));
        lane_started[op.lane] = true;
      }
    }
    if (events) YB_CUDA_CHECK(cudaEventRecord(events[i], s));
    switch (op.type) {
      case OP_CONV: {
        if (i == 0 && e->has_stem_tc) {
          rc = launch_stem_f16(in, in_dtype, B, e->cfg.height, e->cfg.width, op.w_f16, op.bias,
                               make_view(e, op.out), s, e->src_h, e->src_w);
          if (rc) return rc;
          input_converted = true;  // the stem reads the caller's NCHW tensor directly
          break;
        }
        if (!input_converted) {
          rc = launch_input_to_nhwc<T>(in, in_dtype, make_view(e, e->input_nhwc), B, s, e->src_h, e->src_w);
          if (rc) return rc;
          input_converted = true;
        }
        if (op.absorbed) break;
        if (op.bneck) {
          rc = tc_bneck_launch(op.bneck, B, e->tile_ctr ? e->tile_ctr + i : nullptr, s);
        } else if (op.use_tc) {
          rc = tc_conv_launch(op.fold ? op.fold : op.plan, B, out_pred, e->tile_ctr ? e->tile_ctr + i : nullptr, s);
        } else {
          rc = launch_conv_generic<T>(conv_params(e, op, B), s);
        }
        if (rc) return rc;
        break;
      }
      case OP_DWCONV:
        rc = launch_dwconv3x3<T>(conv_params(e, op, B), s);
        if (rc) return rc;
        break;
      case OP_POOL:
        rc = launch_sppf_pool<T>(make_view(e, op.in), make_view(e, op.out), make_view(e, op.out2),
                                 make_view(e, op.out3), B, s);
        if (rc) return rc;
        break;
      case OP_UPSAMPLE:
        rc = launch_upsample2x<T>(make_view(e, op.in), make_view(e, op.out), B, s);
        if (rc) return rc;
        break;
      case OP_DECODE: {
        if (op.fused) break;
        View coef = make_view(e, op.coef);
        rc = launch_decode_level<T>(make_view(e, op.in), make_view(e, op.cls), op.coef.buf >= 0 ? &coef : nullptr, B,
                                    e->cfg.nc, 32, e->cfg.reg_max, op.stride, op.a0, e->A, e->pred_c, out_pred, s);
        if (rc) return rc;
        break;
      }
      case OP_PIXSHUF:
        rc = launch_pixel_shuffle2<T>(make_view(e, op.in), make_view(e, op.out), B, s);
        if (rc) return rc;
        break;
      case OP_ATTN:
        rc = launch_attention<T>(make_view(e, op.in), make_view(e, op.out), make_view(e, op.out2), B, op.nh, op.kd,
                                 op.hd, op.scale, s);
        if (rc) return rc;
        break;
      case OP_PROTO_OUT:
        if (out_proto) {
          rc = launch_proto_out<T>(make_view(e, op.in), out_proto, B, s);
          if (rc) return rc;
        }
        break;
      default:
        set_error("op type not implemented: " + op.name);
        return YB_ERR_NOT_IMPLEMENTED;
    }
    if (lanes && op.feat_level >= 0) YB_CUDA_CHECK(cudaEventRecord(e->ev_feat[op.feat_level], main_s));
    if (lanes && op.fork_id >= 0) YB_CUDA_CHECK(cudaEventRecord(e->ev_fork[op.fork_id], s));
  }
  s = main_s;
  if (lanes)
    for (int l = 1; l < yb_engine::kLanes; l++)
      if (lane_started[l]) {
        YB_CUDA_CHECK(cudaEventRecord(e->ev_done[l], e->side[l]));
        YB_CUDA_CHECK(cudaStreamWaitEvent(main_s, e->ev_done[l], 0));
      }
  if (events) YB_CUDA_CHECK(cudaEventRecord(events[e->ops.size()], s));
  return 0;
}

bool have_device(const char* who, int* ndev) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    set_error(std::string(who) + ": no CUDA device (this library has no CPU fallback)");
    return false;
  }
  if (ndev) *ndev = n;
  return true;
}

}  // namespace yb

// ------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------
extern "C" {

int32_t yb_abi_version(void) { return YB_ABI_VERSION; }

const char* yb_build_info(void) {
  return "yolob200 (sm_90a; wgmma+TMA conv, CUDA-core fp32 parity path) built " __DATE__ " " __TIME__;
}

const char* yb_last_error(void) { return g_last_error.c_str(); }

int32_t yb_create(const yb_config* cfg, yb_engine** out) {
  if (!cfg || !out) { set_error("yb_create: null argument"); return YB_ERR_INVALID_ARG; }
  *out = nullptr;
  if (cfg->arch != YB_ARCH_V8 && cfg->arch != YB_ARCH_V11) { set_error("yb_create: arch must be 8 or 11"); return YB_ERR_INVALID_ARG; }
  if (cfg->size < 0 || cfg->size > 4) { set_error("yb_create: size must be 0..4 (n,s,m,l,x)"); return YB_ERR_INVALID_ARG; }
  if (cfg->task != YB_TASK_DETECT && cfg->task != YB_TASK_SEGMENT) { set_error("yb_create: unsupported task"); return YB_ERR_NOT_IMPLEMENTED; }
  if (cfg->nc <= 0 || cfg->nc >= 4096 || cfg->reg_max != 16) { set_error("yb_create: need 0 < nc < 4096 and reg_max == 16"); return YB_ERR_INVALID_ARG; }
  if (cfg->height <= 0 || cfg->width <= 0 || cfg->height % 32 || cfg->width % 32) { set_error("yb_create: height/width must be positive multiples of 32"); return YB_ERR_INVALID_ARG; }
  if (cfg->max_batch <= 0) { set_error("yb_create: max_batch must be positive"); return YB_ERR_INVALID_ARG; }
  if (cfg->precision != YB_PREC_F32 && cfg->precision != YB_PREC_F16) { set_error("yb_create: bad precision"); return YB_ERR_INVALID_ARG; }
  if (cfg->flags & YB_FLAG_DRY_RUN) {
    std::unique_ptr<yb_engine> d(new yb_engine());
    d->cfg = *cfg;
    d->esize = cfg->precision == YB_PREC_F16 ? 2 : 4;
    int rc = build_graph(d.get());
    if (rc) return rc;
    *out = d.release();
    return YB_OK;
  }
  int ndev = 0;
  if (!have_device("yb_create", &ndev)) return YB_ERR_NO_DEVICE;
  if (cfg->device < 0 || cfg->device >= ndev) { set_error("yb_create: bad device ordinal"); return YB_ERR_INVALID_ARG; }
  YB_CUDA_CHECK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  YB_CUDA_CHECK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) {
    set_error(std::string("yb_create: device '") + prop.name + "' is not sm_90 (Hopper H100); this library only contains sm_90a code");
    return YB_ERR_NO_DEVICE;
  }
  std::unique_ptr<yb_engine> e(new yb_engine());
  e->cfg = *cfg;
  e->esize = cfg->precision == YB_PREC_F16 ? 2 : 4;
  int rc = build_graph(e.get());
  if (rc) return rc;
  // workspace: one arena, every buffer sized for max_batch, 1 KiB aligned (TMA / wgmma friendly)
  size_t off = 0;
  for (auto& b : e->bufs) {
    b.offset = off;
    size_t bytes = (size_t)cfg->max_batch * b.H * b.W * b.C * e->esize;
    off += (bytes + 1023) / 1024 * 1024;
  }
  e->arena_bytes = off;
  YB_CUDA_CHECK(cudaMalloc((void**)&e->arena, off));
  YB_CUDA_CHECK(cudaMemset(e->arena, 0, off));
  YB_CUDA_CHECK(cudaMalloc((void**)&e->tile_ctr, e->ops.size() * sizeof(int)));
  // forward kernels are captured at the highest stream priority: when the caller overlaps post-processing of the
  // previous batch (NMS on another stream) with this forward, freed SMs go to the forward's CTAs first
  int prio_least = 0, prio_greatest = 0;
  YB_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
  YB_CUDA_CHECK(cudaStreamCreateWithPriority(&e->capture_stream, cudaStreamNonBlocking, prio_greatest));
  for (int l = 1; l < yb_engine::kLanes; l++) {
    YB_CUDA_CHECK(cudaStreamCreateWithPriority(&e->side[l], cudaStreamNonBlocking, prio_greatest));
    YB_CUDA_CHECK(cudaEventCreateWithFlags(&e->ev_done[l], cudaEventDisableTiming));
  }
  for (int l = 0; l < 3; l++) {
    YB_CUDA_CHECK(cudaEventCreateWithFlags(&e->ev_feat[l], cudaEventDisableTiming));
    YB_CUDA_CHECK(cudaEventCreateWithFlags(&e->ev_fork[l], cudaEventDisableTiming));
  }
  *out = e.release();
  return YB_OK;
}

void yb_destroy(yb_engine* e) {
  if (!e) return;
  if (e->cfg.flags & YB_FLAG_DRY_RUN) { delete e; return; }
  cudaSetDevice(e->cfg.device);
  for (auto& kv : e->graphs) cudaGraphExecDestroy(kv.second);
  for (auto& op : e->ops) if (op.bneck) tc_bneck_plan_destroy(op.bneck);
  for (auto& op : e->ops) if (op.fold) tc_conv_plan_destroy(op.fold);
  for (auto& op : e->ops) if (op.plan) tc_conv_plan_destroy(op.plan);
  for (void* p : e->dev_allocs) cudaFree(p);
  if (e->arena) cudaFree(e->arena);
  if (e->tile_ctr) cudaFree(e->tile_ctr);
  for (auto& st : e->stage) {
    if (st.in) cudaFree(st.in);
    if (st.pred) cudaFree(st.pred);
    if (st.dets) cudaFree(st.dets);
    if (st.counts) cudaFree(st.counts);
    if (st.proto) cudaFree(st.proto);
    if (st.masks) cudaFree(st.masks);
    if (st.stream) cudaStreamDestroy(st.stream);
  }
  if (e->arena_free) cudaEventDestroy(e->arena_free);
  if (e->capture_stream) cudaStreamDestroy(e->capture_stream);
  for (int l = 1; l < yb_engine::kLanes; l++) {
    if (e->side[l]) cudaStreamDestroy(e->side[l]);
    if (e->ev_done[l]) cudaEventDestroy(e->ev_done[l]);
  }
  for (int l = 0; l < 3; l++) {
    if (e->ev_feat[l]) cudaEventDestroy(e->ev_feat[l]);
    if (e->ev_fork[l]) cudaEventDestroy(e->ev_fork[l]);
  }
  delete e;
}

int32_t yb_num_anchors(const yb_engine* e) { return e ? e->A : 0; }
int32_t yb_pred_channels(const yb_engine* e) { return e ? e->pred_c : 0; }
int32_t yb_num_expected_tensors(const yb_engine* e) { return e ? (int32_t)e->expected.size() : 0; }
const char* yb_expected_tensor_name(const yb_engine* e, int32_t i) {
  if (!e || i < 0 || i >= (int32_t)e->expected.size()) return nullptr;
  return e->expected[i].c_str();
}

int32_t yb_load_tensor(yb_engine* e, const char* name, int32_t dtype, int32_t ndim, const int64_t* shape,
                       const void* data) {
  if (!e || !name || (ndim > 0 && !shape) || ndim < 0 || ndim > 8) { set_error("yb_load_tensor: bad argument"); return YB_ERR_INVALID_ARG; }
  if (e->finalized) { set_error("yb_load_tensor: weights already finalized"); return YB_ERR_STATE; }
  int64_t n = 1;
  for (int i = 0; i < ndim; i++) {
    if (shape[i] < 0) { set_error("yb_load_tensor: negative dimension"); return YB_ERR_INVALID_ARG; }
    n *= shape[i];
  }
  if (n > 0 && !data) { set_error("yb_load_tensor: null data"); return YB_ERR_INVALID_ARG; }
  HostTensor t;
  t.shape.assign(shape, shape + ndim);
  t.data.resize((size_t)n);
  switch (dtype) {
    case YB_F32:
      std::memcpy(t.data.data(), data, (size_t)n * 4);
      break;
    case YB_F16: {
      const __half* h = reinterpret_cast<const __half*>(data);
      for (int64_t i = 0; i < n; i++) t.data[i] = __half2float(h[i]);
      break;
    }
    case YB_BF16: {
      const uint16_t* h = reinterpret_cast<const uint16_t*>(data);
      for (int64_t i = 0; i < n; i++) {
        uint32_t u = (uint32_t)h[i] << 16;
        std::memcpy(&t.data[i], &u, 4);
      }
      break;
    }
    default:
      set_error("yb_load_tensor: unsupported dtype " + std::to_string(dtype) + " (5=f16, 6=f32, 15=bf16)");
      return YB_ERR_INVALID_ARG;
  }
  e->host[name] = std::move(t);
  return YB_OK;
}

// true when no op other than ops[i] and ops[i + 1] reads or writes buffer `buf` (the fusion passes of yb_finalize_weights)
static bool only_pair_uses(const yb_engine* e, size_t i, int buf) {
  for (size_t j = 0; j < e->ops.size(); j++) {
    if (j == i || j == i + 1) continue;
    const OpDesc& o = e->ops[j];
    for (const VRef* r : {&o.in, &o.out, &o.res, &o.out2, &o.out3, &o.cls, &o.coef})
      if (r->buf == buf) return false;
  }
  return true;
}

int32_t yb_finalize_weights(yb_engine* e) {
  if (!e) { set_error("yb_finalize_weights: null engine"); return YB_ERR_INVALID_ARG; }
  if (e->finalized) { set_error("yb_finalize_weights: already finalized"); return YB_ERR_STATE; }
  if (e->cfg.flags & YB_FLAG_DRY_RUN) { set_error("yb_finalize_weights: dry-run engine has no device"); return YB_ERR_STATE; }
  YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
  const bool f16 = e->cfg.precision == YB_PREC_F16;
  const bool allow_tc = f16 && !(e->cfg.flags & YB_FLAG_NO_TCGEN05);
  if (allow_tc) {
    // Detect tail fusion: when every final 1x1 conv of a level can run on the tensor-core kernel, their
    // epilogues write the prediction tensor directly and the decode kernel is dropped.
    for (auto& d : e->ops) {
      if (d.type != OP_DECODE) continue;
      std::vector<OpDesc*> prod;
      bool ok = true;
      for (int bufid : {d.in.buf, d.cls.buf, d.coef.buf}) {
        if (bufid < 0) continue;
        OpDesc* pr = nullptr;
        for (auto& c : e->ops)
          if (c.type == OP_CONV && c.out.buf == bufid) pr = &c;
        if (!pr || pr->k != 1 || pr->s != 1 || pr->cin % 16 || pr->cout % 16 || pr->cout > 256) ok = false;
        prod.push_back(pr);
      }
      if (!ok || e->cfg.reg_max != 16) continue;
      const BufDesc& lb = e->bufs[d.in.buf];
      for (OpDesc* pr : prod) {
        EpiDecode& dc = pr->dec;
        dc.A = e->A; dc.Ctot = e->pred_c; dc.a0 = d.a0; dc.Wl = lb.W; dc.HW = lb.H * lb.W; dc.stride = d.stride;
        if (pr->out.buf == d.in.buf) { dc.mode = EPI_DFL_BOX; dc.ch0 = 0; }
        else if (pr->out.buf == d.cls.buf) { dc.mode = EPI_SIGMOID; dc.ch0 = 4; }
        else { dc.mode = EPI_RAW; dc.ch0 = 4 + e->cfg.nc; }
      }
      d.fused = true;
    }
  }
  for (size_t i = 0; i < e->ops.size(); i++) {
    OpDesc& op = e->ops[i];
    if (op.type != OP_CONV && op.type != OP_DWCONV) continue;
    int rc = finalize_conv(e, op);
    if (rc) return rc;
    if (op.type == OP_CONV && allow_tc) {
      if (i == 0) {
        e->has_stem_tc = true;  // Cin = 3: dedicated stem kernel reading NCHW directly
        continue;
      }
      ConvParams p = conv_params(e, op, e->cfg.max_batch);
      p.w = op.w_f16;
      p.dec = op.dec;
      p.share_sms = (op.lane > 0 && !(e->cfg.flags & YB_FLAG_NO_CONCURRENCY)) ? 1 : 0;
      if (tc_conv_supported(p)) {
        std::string err;
        op.plan = tc_conv_plan_create(p, &err);
        if (!op.plan) { set_error("tensor-core plan failed for " + op.name + ": " + err); return YB_ERR_CUDA; }
        op.use_tc = true;
        if (getenv("YB_DEBUG_PLANS")) fprintf(stderr, "[plan] %-30s k%d s%d %4d->%4d @%dx%d  %s\n", op.name.c_str(), op.k, op.s, op.cin, op.cout,
                                              p.Ho, p.Wo, tc_conv_plan_describe(op.plan).c_str());
      }
    }
  }
  for (auto& d : e->ops) {
    if (d.type != OP_DECODE || !d.fused) continue;
    for (auto& c : e->ops)
      if (c.type == OP_CONV && c.dec.mode != EPI_STORE && c.dec.a0 == d.a0 && !c.use_tc) {
        set_error("internal: fused decode producer " + c.name + " did not get a tensor-core plan");
        return YB_ERR_STATE;
      }
  }
  // Bottleneck fusion: a 3x3 s1 tensor-core conv whose output buffer has exactly one reader, the next 3x3 s1 conv of the
  // same lane, runs inside that conv's launch (tc_bneck_plan_create decides whether the pair fits).  The first op stays in
  // the op list, launches nothing and keeps its arena buffer for yb_debug_read_activation.
  for (size_t i = 1; i + 1 < e->ops.size(); i++) {
    OpDesc &a = e->ops[i], &b = e->ops[i + 1];
    if (a.type != OP_CONV || b.type != OP_CONV || !a.use_tc || !b.use_tc || a.absorbed || a.bneck) continue;
    if (a.k != 3 || a.s != 1 || b.k != 3 || b.s != 1 || a.lane != b.lane) continue;
    if (b.in.buf != a.out.buf || b.in.coff != a.out.coff || b.in.C != a.out.C) continue;
    if (!only_pair_uses(e, i, a.out.buf) || b.res.buf == a.out.buf) continue;
    std::string err;
    b.bneck = tc_bneck_plan_create(a.plan, b.plan, &err);
    if (!b.bneck) continue;
    a.absorbed = true;
    if (getenv("YB_DEBUG_PLANS")) fprintf(stderr, "[plan] %-30s %s (absorbs %s)\n", b.name.c_str(), tc_bneck_plan_describe(b.bneck).c_str(), a.name.c_str());
  }
  // 1x1 fold: a tensor-core conv that stores its output, whose output buffer has exactly one reader, the next op of the
  // same lane, a 1x1 s1 tensor-core conv: that 1x1 runs inside the conv's launch on the accumulator registers of each
  // tile (tc_fold_plan_create decides whether the pair fits).  The producer stays in the op list, launches nothing and
  // keeps its arena buffer for yb_debug_read_activation.  YB_NO_FOLD1X1=1 turns the pass off.
  const char* no_fold = getenv("YB_NO_FOLD1X1");
  for (size_t i = 1; i + 1 < e->ops.size() && !(no_fold && atoi(no_fold)); i++) {
    OpDesc &a = e->ops[i], &b = e->ops[i + 1];
    if (a.type != OP_CONV || b.type != OP_CONV || !a.use_tc || !b.use_tc || a.absorbed || a.bneck || a.fold || b.bneck) continue;
    if (a.res.buf >= 0 || a.dec.mode != EPI_STORE || b.k != 1 || b.s != 1 || b.res.buf >= 0 || a.lane != b.lane) continue;
    if (b.in.buf != a.out.buf || b.in.coff != a.out.coff || b.in.C != a.out.C) continue;
    if (!only_pair_uses(e, i, a.out.buf)) continue;
    std::string err;
    b.fold = tc_fold_plan_create(a.plan, b.plan, &err);
    if (!b.fold) {
      if (getenv("YB_DEBUG_PLANS")) fprintf(stderr, "[plan] %-30s fold refused (%s): %s\n", b.name.c_str(), a.name.c_str(), err.c_str());
      continue;
    }
    a.absorbed = a.folded = true;
    if (getenv("YB_DEBUG_PLANS")) fprintf(stderr, "[plan] %-30s %s (folds %s)\n", b.name.c_str(), tc_conv_plan_describe(b.fold).c_str(), a.name.c_str());
  }
  e->lanes_ok = allow_tc && !(e->cfg.flags & YB_FLAG_NO_CONCURRENCY);
  for (auto& d : e->ops)
    if (d.type == OP_DECODE && !d.fused) e->lanes_ok = false;  // the generic decode kernel joins box+cls lanes
  e->host.clear();
  e->finalized = true;
  return YB_OK;
}

int32_t yb_forward(yb_engine* e, const void* in, int32_t in_dtype, int32_t batch, float* out_pred,
                   float* out_proto, void* stream) {
  if (!e) { set_error("yb_forward: null argument"); return YB_ERR_INVALID_ARG; }
  return yb_forward_padded(e, in, in_dtype, batch, e->cfg.height, e->cfg.width, out_pred, out_proto, stream);
}

int32_t yb_forward_padded(yb_engine* e, const void* in, int32_t in_dtype, int32_t batch, int32_t src_height, int32_t src_width,
                          float* out_pred, float* out_proto, void* stream) {
  if (!e || !in || !out_pred) { set_error("yb_forward: null argument"); return YB_ERR_INVALID_ARG; }
  if (src_height <= 0 || src_width <= 0 || src_height > e->cfg.height || src_width > e->cfg.width) {
    set_error("yb_forward_padded: source size must be within the planned input size");
    return YB_ERR_INVALID_ARG;
  }
  e->src_h = src_height; e->src_w = src_width;
  if (!e->finalized) { set_error("yb_forward: call yb_finalize_weights first"); return YB_ERR_STATE; }
  if (batch <= 0 || batch > e->cfg.max_batch) { set_error("yb_forward: batch outside [1, max_batch]"); return YB_ERR_INVALID_ARG; }
  if (in_dtype != YB_U8 && in_dtype != YB_F16 && in_dtype != YB_F32) { set_error("yb_forward: in_dtype must be u8/f16/f32"); return YB_ERR_INVALID_ARG; }
  if (e->cfg.task == YB_TASK_SEGMENT && !out_proto) { set_error("yb_forward: segment engine needs out_proto"); return YB_ERR_INVALID_ARG; }
  YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const bool f16 = e->cfg.precision == YB_PREC_F16;
  auto run = [&](cudaStream_t st) {
    return f16 ? run_ops<__half>(e, in, in_dtype, batch, out_pred, out_proto, st)
               : run_ops<float>(e, in, in_dtype, batch, out_pred, out_proto, st);
  };
  if (e->cfg.flags & YB_FLAG_NO_GRAPH) return run(s);
  yb_engine::GraphKey key{in, in_dtype, batch, out_pred, out_proto, src_height, src_width};
  auto it = e->graphs.find(key);
  if (it != e->graphs.end()) {
    YB_CUDA_CHECK(cudaGraphLaunch(it->second, s));
    return YB_OK;
  }
  // first call with these buffers runs eagerly (also performs one-time attribute setup); the
  // second call captures the launch sequence on a private stream and replays it from then on
  if (e->seen[key]++ == 0) return run(s);
  cudaGraph_t graph = nullptr;
  YB_CUDA_CHECK(cudaStreamBeginCapture(e->capture_stream, cudaStreamCaptureModeThreadLocal));
  int rc = run(e->capture_stream);
  cudaError_t ce = cudaStreamEndCapture(e->capture_stream, &graph);
  if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
  if (ce != cudaSuccess) { set_error(std::string("graph capture failed: ") + cudaGetErrorString(ce)); return YB_ERR_CUDA; }
  cudaGraphExec_t exec = nullptr;
  ce = cudaGraphInstantiate(&exec, graph, 0);
  cudaGraphDestroy(graph);
  if (ce != cudaSuccess) { set_error(std::string("graph instantiate failed: ") + cudaGetErrorString(ce)); return YB_ERR_CUDA; }
  if (e->graphs.size() > 64) {  // bound the cache
    for (auto& kv : e->graphs) cudaGraphExecDestroy(kv.second);
    e->graphs.clear();
  }
  e->graphs[key] = exec;
  YB_CUDA_CHECK(cudaGraphLaunch(exec, s));
  return YB_OK;
}

int32_t yb_nms(const float* pred, int32_t batch, int32_t channels, int32_t anchors, int32_t nc, float conf_thres,
               float iou_thres, int32_t max_det, int32_t max_nms, int32_t max_wh, float* dets, int32_t* counts,
               int32_t* keep_idx, void* stream) {
  if (!pred || !dets || !counts) { set_error("yb_nms: null argument"); return YB_ERR_INVALID_ARG; }
  return nms_launch(pred, batch, channels, anchors, nc, conf_thres, iou_thres, max_det, max_nms, max_wh, dets, counts,
                    keep_idx, (cudaStream_t)stream);
}

int32_t yb_masks(const float* proto, const float* dets, const int32_t* counts, int32_t batch, int32_t max_det,
                 int32_t nm, int32_t mh, int32_t mw, int32_t height, int32_t width, uint8_t* masks, void* stream) {
  if (!proto || !dets || !counts || !masks) { set_error("yb_masks: null argument"); return YB_ERR_INVALID_ARG; }
  if (batch <= 0 || max_det <= 0 || nm <= 0 || mh <= 0 || mw <= 0 || height <= 0 || width <= 0) { set_error("yb_masks: bad shape"); return YB_ERR_INVALID_ARG; }
  return masks_launch(proto, dets, counts, batch, max_det, nm, mh, mw, height, width, masks, (cudaStream_t)stream);
}

int32_t yb_detection_loss(const float* boxes, const float* scores, int32_t batch, int32_t nc, int32_t reg_max,
                          int32_t height, int32_t width, const float* targets_host, int32_t n_targets, int32_t topk,
                          float hyp_box, float hyp_cls, float hyp_dfl, float* loss_items, float* grad_boxes,
                          float* grad_scores, uint8_t* fg, int32_t* gt_idx, float* target_score, void* stream) {
  if (!boxes || !scores || !loss_items || (n_targets > 0 && !targets_host)) {
    set_error("yb_detection_loss: null argument");
    return YB_ERR_INVALID_ARG;
  }
  if (!have_device("yb_detection_loss")) return YB_ERR_NO_DEVICE;
  return detection_loss_launch(boxes, scores, batch, nc, reg_max, height, width, targets_host, n_targets, topk, hyp_box,
                               hyp_cls, hyp_dfl, loss_items, grad_boxes, grad_scores, fg, gt_idx, target_score,
                               (cudaStream_t)stream);
}

int32_t yb_bn_silu_train_forward(const float* z, int64_t rows, int32_t channels, int32_t pitch, const float* gamma,
                                 const float* beta, float eps, float momentum, int32_t act, float* running_mean,
                                 float* running_var, float* y, int32_t ypitch, float* save_mean, float* save_invstd,
                                 void* stream) {
  if (!z || !gamma || !beta || !y || !save_mean || !save_invstd || (!running_mean) != (!running_var)) {
    set_error("yb_bn_silu_train_forward: null argument");
    return YB_ERR_INVALID_ARG;
  }
  if (!have_device("yb_bn_silu_train_forward")) return YB_ERR_NO_DEVICE;
  return bn_silu_train_forward(z, rows, channels, pitch, gamma, beta, eps, momentum, act, running_mean, running_var, y, ypitch,
                               save_mean, save_invstd, (cudaStream_t)stream);
}

int32_t yb_bn_silu_backward(const float* z, const float* dy, int64_t rows, int32_t channels, int32_t pitch,
                            int32_t dpitch, const float* gamma, const float* beta, const float* save_mean,
                            const float* save_invstd, int32_t act, float* dz, int32_t zpitch, float* dgamma,
                            float* dbeta, void* stream) {
  if (!z || !dy || !gamma || !beta || !save_mean || !save_invstd || !dz || !dgamma || !dbeta) {
    set_error("yb_bn_silu_backward: null argument");
    return YB_ERR_INVALID_ARG;
  }
  if (!have_device("yb_bn_silu_backward")) return YB_ERR_NO_DEVICE;
  return bn_silu_backward(z, dy, rows, channels, pitch, dpitch, gamma, beta, save_mean, save_invstd, act, dz, zpitch, dgamma,
                          dbeta, (cudaStream_t)stream);
}

int32_t yb_adamw_step(float* p, const float* g, float* m, float* v, int64_t n, int32_t step, float lr, float beta1,
                      float beta2, float eps, float weight_decay, void* stream) {
  if (!p || !g || !m || !v) {
    set_error("yb_adamw_step: null argument");
    return YB_ERR_INVALID_ARG;
  }
  if (!have_device("yb_adamw_step")) return YB_ERR_NO_DEVICE;
  return adamw_step(p, g, m, v, n, step, lr, beta1, beta2, eps, weight_decay, (cudaStream_t)stream);
}

int32_t yb_conv_forward_f32(const float* x, const float* w_packed, const float* bias, int32_t n, int32_t height,
                            int32_t width, int32_t cin, int32_t cout, int32_t k, int32_t stride, int32_t pad, float* z,
                            void* stream) {
  if (!x || !w_packed || !z) { set_error("yb_conv_forward_f32: null argument"); return YB_ERR_INVALID_ARG; }
  if (n <= 0 || height <= 0 || width <= 0 || cin <= 0 || cout <= 0 || k <= 0 || stride <= 0 || pad < 0) {
    set_error("yb_conv_forward_f32: bad shape");
    return YB_ERR_SHAPE;
  }
  if (!have_device("yb_conv_forward_f32")) return YB_ERR_NO_DEVICE;
  static float* zero_bias = nullptr;  // the generic kernel always adds a bias vector
  static int zero_cap = 0;
  if (!bias && zero_cap < cout) {
    if (zero_bias) cudaFree(zero_bias);
    zero_cap = std::max(cout, 4096);
    YB_CUDA_CHECK(cudaMalloc((void**)&zero_bias, (size_t)zero_cap * sizeof(float)));
    YB_CUDA_CHECK(cudaMemset(zero_bias, 0, (size_t)zero_cap * sizeof(float)));
  }
  ConvParams p;
  p.in.base = const_cast<float*>(x); p.in.H = height; p.in.W = width; p.in.pitch = cin; p.in.coff = 0; p.in.C = cin;
  p.Ho = (height + 2 * pad - k) / stride + 1;
  p.Wo = (width + 2 * pad - k) / stride + 1;
  p.out.base = z; p.out.H = p.Ho; p.out.W = p.Wo; p.out.pitch = cout; p.out.coff = 0; p.out.C = cout;
  p.w = w_packed;
  p.bias = bias ? bias : zero_bias;
  p.B = n; p.Cin = cin; p.Cout = cout; p.k = k; p.stride = stride; p.pad = pad;
  p.act = ACT_NONE;
  return launch_conv_generic<float>(p, (cudaStream_t)stream);
}

int32_t yb_conv_backward_data(const float* dz, const float* w, int32_t n, int32_t height, int32_t width, int32_t cin,
                              int32_t cout, int32_t k, int32_t stride, int32_t pad, float* dx, void* stream) {
  if (!dz || !w || !dx) { set_error("yb_conv_backward_data: null argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_conv_backward_data")) return YB_ERR_NO_DEVICE;
  return conv_backward_data(dz, w, n, height, width, cin, cout, k, stride, pad, dx, (cudaStream_t)stream);
}

int32_t yb_conv_backward_weight(const float* x, const float* dz, int32_t n, int32_t height, int32_t width, int32_t cin,
                                int32_t cout, int32_t k, int32_t stride, int32_t pad, float* dw, void* stream) {
  if (!x || !dz || !dw) { set_error("yb_conv_backward_weight: null argument"); return YB_ERR_INVALID_ARG; }
  if (!have_device("yb_conv_backward_weight")) return YB_ERR_NO_DEVICE;
  return conv_backward_weight(x, dz, n, height, width, cin, cout, k, stride, pad, dw, (cudaStream_t)stream);
}

static int32_t predict_enqueue(yb_engine* e, yb_engine::Stage& st, const uint8_t* images_host, int32_t batch,
                               float conf_thres, float iou_thres, int32_t max_det, float* dets_host,
                               int32_t* counts_host, cudaStream_t s, const char* who, yb_comm* comm = nullptr,
                               int comm_slot = 0, uint8_t* masks_host = nullptr, int32_t mask_cap = 0) {
  if (!e || !images_host || !dets_host || !counts_host) { set_error(std::string(who) + ": null argument"); return YB_ERR_INVALID_ARG; }
  if (!e->finalized) { set_error(std::string(who) + ": call yb_finalize_weights first"); return YB_ERR_STATE; }
  if (batch <= 0 || batch > e->cfg.max_batch) { set_error(std::string(who) + ": batch outside [1, max_batch]"); return YB_ERR_INVALID_ARG; }
  const bool seg = e->cfg.task == YB_TASK_SEGMENT;
  if (seg != (masks_host != nullptr)) { set_error(std::string(who) + (seg ? ": segment engines go through yb_predict_seg_u8_submit" : ": masks requested from a detect engine")); return YB_ERR_INVALID_ARG; }
  if (seg && (comm || mask_cap <= 0 || mask_cap > max_det)) { set_error(std::string(who) + ": need 0 < mask_cap <= max_det (and no exchange) for segment engines"); return YB_ERR_INVALID_ARG; }
  if (max_det <= 0 || max_det > 1024) { set_error(std::string(who) + ": max_det outside [1,1024]"); return YB_ERR_INVALID_ARG; }
  YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
  const size_t img_bytes = (size_t)3 * e->cfg.height * e->cfg.width;
  const int row_w = 6 + (e->pred_c - 4 - e->cfg.nc);
  if (!st.in) {
    YB_CUDA_CHECK(cudaMalloc((void**)&st.in, img_bytes * e->cfg.max_batch));
    YB_CUDA_CHECK(cudaMalloc((void**)&st.pred, (size_t)e->cfg.max_batch * e->pred_c * e->A * sizeof(float)));
    YB_CUDA_CHECK(cudaMalloc((void**)&st.counts, (size_t)e->cfg.max_batch * sizeof(int)));
  }
  if (st.max_det < max_det) {
    if (st.dets) cudaFree(st.dets);
    st.dets = nullptr;
    YB_CUDA_CHECK(cudaMalloc((void**)&st.dets, (size_t)e->cfg.max_batch * max_det * row_w * sizeof(float)));
    st.max_det = max_det;
  }
  YB_CUDA_CHECK(cudaMemcpyAsync(st.in, images_host, img_bytes * batch, cudaMemcpyHostToDevice, s));
  // one activation arena per engine: forwards of different slots are serialised on the device (their H2D
  // copies, NMS and D2H copies still overlap the other slot's forward)
  if (!e->arena_free) YB_CUDA_CHECK(cudaEventCreateWithFlags(&e->arena_free, cudaEventDisableTiming));
  if (e->arena_used) YB_CUDA_CHECK(cudaStreamWaitEvent(s, e->arena_free, 0));
  const int mh = e->cfg.height / 4, mw = e->cfg.width / 4;
  if (seg) {
    if (!st.proto) YB_CUDA_CHECK(cudaMalloc((void**)&st.proto, (size_t)e->cfg.max_batch * 32 * mh * mw * sizeof(float)));
    if (st.mask_cap < mask_cap) {
      if (st.masks) cudaFree(st.masks);
      st.masks = nullptr;
      YB_CUDA_CHECK(cudaMalloc((void**)&st.masks, (size_t)e->cfg.max_batch * mask_cap * e->cfg.height * e->cfg.width));
      st.mask_cap = mask_cap;
    }
  }
  int rc = yb_forward(e, st.in, YB_U8, batch, st.pred, seg ? st.proto : nullptr, (void*)s);
  if (rc) return rc;
  YB_CUDA_CHECK(cudaEventRecord(e->arena_free, s));
  e->arena_used = true;
  if (comm) {
    // multi-GPU: NMS writes its rows + counts straight into the exchange's send buffer; every rank's payload is
    // pushed into every rank's window over NVLink (csrc/comm.cu), then ONE strided D2H copy per array brings the
    // detections of ALL ranks (global image order = rank order) to the host
    int32_t world = 1;
    int64_t cbytes = 0;
    yb_comm_info(comm, nullptr, &world, &cbytes, nullptr);
    const size_t dets_bytes = ((size_t)batch * max_det * row_w * sizeof(float) + 15) / 16 * 16;
    if ((int64_t)(dets_bytes + ((size_t)batch * 4 + 15) / 16 * 16) > cbytes) {
      set_error(std::string(who) + ": detection payload larger than the exchange's bytes_per_rank");
      return YB_ERR_INVALID_ARG;
    }
    char* send = (char*)yb_comm_send_buffer(comm, comm_slot);
    const char* win = (const char*)yb_comm_window(comm, comm_slot);
    if (!send || !win) { set_error(std::string(who) + ": bad exchange slot"); return YB_ERR_INVALID_ARG; }
    rc = nms_launch(st.pred, batch, e->pred_c, e->A, e->cfg.nc, conf_thres, iou_thres, max_det, 30000, 7680,
                    (float*)send, (int*)(send + dets_bytes), nullptr, s);
    if (rc) return rc;
    rc = yb_comm_allgather(comm, comm_slot, (void*)s);
    if (rc) return rc;
    const size_t dw = (size_t)batch * max_det * row_w * sizeof(float);
    YB_CUDA_CHECK(cudaMemcpy2DAsync(dets_host, dw, win, (size_t)cbytes, dw, world, cudaMemcpyDeviceToHost, s));
    YB_CUDA_CHECK(cudaMemcpy2DAsync(counts_host, (size_t)batch * 4, win + dets_bytes, (size_t)cbytes, (size_t)batch * 4, world,
                                    cudaMemcpyDeviceToHost, s));
    return yb_comm_release(comm, comm_slot, (void*)s);
  }
  rc = nms_launch(st.pred, batch, e->pred_c, e->A, e->cfg.nc, conf_thres, iou_thres, max_det, 30000, 7680, st.dets,
                  st.counts, nullptr, s);
  if (rc) return rc;
  YB_CUDA_CHECK(cudaMemcpyAsync(dets_host, st.dets, (size_t)batch * max_det * row_w * sizeof(float),
                                cudaMemcpyDeviceToHost, s));
  YB_CUDA_CHECK(cudaMemcpyAsync(counts_host, st.counts, (size_t)batch * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (seg) {
    // Segmenter.cs:54: process_mask(upsample: true) of the kept rows; masks beyond an image's count are left untouched
    rc = masks_launch(st.proto, st.dets, st.counts, batch, max_det, 32, mh, mw, e->cfg.height, e->cfg.width, st.masks, s, mask_cap);
    if (rc) return rc;
    YB_CUDA_CHECK(cudaMemcpyAsync(masks_host, st.masks, (size_t)batch * mask_cap * e->cfg.height * e->cfg.width,
                                  cudaMemcpyDeviceToHost, s));
  }
  return YB_OK;
}

int32_t yb_predict_u8(yb_engine* e, const uint8_t* images_host, int32_t batch, float conf_thres, float iou_thres,
                      int32_t max_det, float* dets_host, int32_t* counts_host, void* stream) {
  if (!e) { set_error("yb_predict_u8: null argument"); return YB_ERR_INVALID_ARG; }
  int rc = predict_enqueue(e, e->stage[0], images_host, batch, conf_thres, iou_thres, max_det, dets_host, counts_host,
                           (cudaStream_t)stream, "yb_predict_u8");
  if (rc) return rc;
  YB_CUDA_CHECK(cudaStreamSynchronize((cudaStream_t)stream));
  return YB_OK;
}

int32_t yb_predict_u8_submit(yb_engine* e, int32_t slot, const uint8_t* images_host, int32_t batch, float conf_thres,
                             float iou_thres, int32_t max_det, float* dets_host, int32_t* counts_host) {
  if (!e || slot < 0 || slot >= yb_engine::kSlots) { set_error("yb_predict_u8_submit: bad engine / slot (0..3)"); return YB_ERR_INVALID_ARG; }
  yb_engine::Stage& st = e->stage[1 + slot];
  if (!st.stream) {
    YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
    YB_CUDA_CHECK(cudaStreamCreateWithFlags(&st.stream, cudaStreamNonBlocking));
  }
  return predict_enqueue(e, st, images_host, batch, conf_thres, iou_thres, max_det, dets_host, counts_host, st.stream,
                         "yb_predict_u8_submit");
}

int32_t yb_predict_u8_submit_gather(yb_engine* e, yb_comm* comm, int32_t slot, const uint8_t* images_host, int32_t batch,
                                    float conf_thres, float iou_thres, int32_t max_det, float* all_dets_host,
                                    int32_t* all_counts_host) {
  if (!e || !comm || slot < 0 || slot >= yb_engine::kSlots) { set_error("yb_predict_u8_submit_gather: bad engine / comm / slot (0..3)"); return YB_ERR_INVALID_ARG; }
  yb_engine::Stage& st = e->stage[1 + slot];
  if (!st.stream) {
    YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
    YB_CUDA_CHECK(cudaStreamCreateWithFlags(&st.stream, cudaStreamNonBlocking));
  }
  return predict_enqueue(e, st, images_host, batch, conf_thres, iou_thres, max_det, all_dets_host, all_counts_host,
                         st.stream, "yb_predict_u8_submit_gather", comm, slot);
}

int32_t yb_predict_seg_u8_submit(yb_engine* e, int32_t slot, const uint8_t* images_host, int32_t batch, float conf_thres,
                                 float iou_thres, int32_t max_det, int32_t mask_cap, float* dets_host, int32_t* counts_host,
                                 uint8_t* masks_host) {
  if (!e || !masks_host || slot < 0 || slot >= yb_engine::kSlots) { set_error("yb_predict_seg_u8_submit: bad engine / masks / slot (0..3)"); return YB_ERR_INVALID_ARG; }
  yb_engine::Stage& st = e->stage[1 + slot];
  if (!st.stream) {
    YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
    YB_CUDA_CHECK(cudaStreamCreateWithFlags(&st.stream, cudaStreamNonBlocking));
  }
  return predict_enqueue(e, st, images_host, batch, conf_thres, iou_thres, max_det, dets_host, counts_host, st.stream,
                         "yb_predict_seg_u8_submit", nullptr, 0, masks_host, mask_cap);
}

int32_t yb_predict_u8_wait(yb_engine* e, int32_t slot) {
  if (!e || slot < 0 || slot >= yb_engine::kSlots) { set_error("yb_predict_u8_wait: bad engine / slot (0..3)"); return YB_ERR_INVALID_ARG; }
  yb_engine::Stage& st = e->stage[1 + slot];
  if (!st.stream) { set_error("yb_predict_u8_wait: nothing was submitted on this slot"); return YB_ERR_STATE; }
  YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
  YB_CUDA_CHECK(cudaStreamSynchronize(st.stream));
  return YB_OK;
}

int32_t yb_num_ops(const yb_engine* e) { return e ? (int32_t)e->ops.size() : 0; }
const char* yb_op_name(const yb_engine* e, int32_t i) {
  if (!e || i < 0 || i >= (int32_t)e->ops.size()) return nullptr;
  return e->ops[i].name.c_str();
}

int32_t yb_debug_read_activation(yb_engine* e, int32_t op_index, int32_t batch, float* host_out, int64_t host_capacity,
                                 int32_t chw[3]) {
  if (!e || !host_out || !chw || op_index < 0 || op_index >= (int32_t)e->ops.size()) { set_error("yb_debug_read_activation: bad argument"); return YB_ERR_INVALID_ARG; }
  YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
  const OpDesc& op = e->ops[op_index];
  if (op.type == OP_DECODE || (op.use_tc && op.dec.mode != EPI_STORE)) {
    set_error("yb_debug_read_activation: op '" + op.name + "' writes the prediction tensor directly (fused head decode)");
    return YB_ERR_STATE;
  }
  View v = make_view(e, op.out);
  chw[0] = v.C; chw[1] = v.H; chw[2] = v.W;
  const int64_t n = (int64_t)batch * v.C * v.H * v.W;
  if (n > host_capacity) { set_error("yb_debug_read_activation: host buffer too small"); return YB_ERR_INVALID_ARG; }
  int rc = 0;
  if (op.absorbed) {
    // The fused Bottleneck (shared memory) or the fold (registers) never stored this op's output: materialise it now into the op's own arena
    // buffer with the fp16 CUDA-core twin (same fp16-rounded weights).  Its input slice is still what the last forward
    // read, because arena buffers are never reused within a forward.
    rc = launch_conv_generic<__half>(conv_params(e, op, batch), 0);
    if (rc) return rc;
  }
  float* d = nullptr;
  YB_CUDA_CHECK(cudaMalloc((void**)&d, n * sizeof(float)));
  rc = e->cfg.precision == YB_PREC_F16 ? launch_view_to_nchw_f32<__half>(v, d, batch, 0)
                                           : launch_view_to_nchw_f32<float>(v, d, batch, 0);
  if (!rc && cudaMemcpy(host_out, d, n * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) {
    set_error("yb_debug_read_activation: copy failed");
    rc = YB_ERR_CUDA;
  }
  cudaFree(d);
  return rc;
}

int32_t yb_profile_forward(yb_engine* e, const void* in, int32_t in_dtype, int32_t batch, float* out_pred,
                           float* out_proto, float* ms_per_op, int32_t n_ops, void* stream) {
  if (!e || !in || !out_pred || !ms_per_op) { set_error("yb_profile_forward: null argument"); return YB_ERR_INVALID_ARG; }
  if (!e->finalized) { set_error("yb_profile_forward: call yb_finalize_weights first"); return YB_ERR_STATE; }
  if (batch <= 0 || batch > e->cfg.max_batch || n_ops < (int32_t)e->ops.size()) { set_error("yb_profile_forward: bad batch / n_ops"); return YB_ERR_INVALID_ARG; }
  YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<cudaEvent_t> ev(e->ops.size() + 1);
  for (auto& x : ev) YB_CUDA_CHECK(cudaEventCreate(&x));
  int rc = e->cfg.precision == YB_PREC_F16 ? run_ops<__half>(e, in, in_dtype, batch, out_pred, out_proto, s, ev.data())
                                           : run_ops<float>(e, in, in_dtype, batch, out_pred, out_proto, s, ev.data());
  if (!rc && cudaStreamSynchronize(s) != cudaSuccess) { set_error("yb_profile_forward: sync failed"); rc = YB_ERR_CUDA; }
  if (!rc)
    for (size_t i = 0; i < e->ops.size(); i++) cudaEventElapsedTime(&ms_per_op[i], ev[i], ev[i + 1]);
  for (auto& x : ev) cudaEventDestroy(x);
  return rc;
}

int32_t yb_time_op(yb_engine* e, int32_t op_index, const void* in, int32_t in_dtype, int32_t batch, float* out_pred,
                   float* out_proto, int32_t reps, float* ms_per_launch, void* stream) {
  if (!e || !in || !out_pred || !ms_per_launch || reps <= 0) { set_error("yb_time_op: bad argument"); return YB_ERR_INVALID_ARG; }
  if (!e->finalized) { set_error("yb_time_op: call yb_finalize_weights first"); return YB_ERR_STATE; }
  if (op_index < 0 || op_index >= (int32_t)e->ops.size() || batch <= 0 || batch > e->cfg.max_batch) { set_error("yb_time_op: bad op / batch"); return YB_ERR_INVALID_ARG; }
  YB_CUDA_CHECK(cudaSetDevice(e->cfg.device));
  cudaStream_t s = (cudaStream_t)stream;
  const bool f16 = e->cfg.precision == YB_PREC_F16;
  auto once = [&]() {
    return f16 ? run_ops<__half>(e, in, in_dtype, batch, out_pred, out_proto, s, nullptr, op_index)
               : run_ops<float>(e, in, in_dtype, batch, out_pred, out_proto, s, nullptr, op_index);
  };
  cudaEvent_t a, b;
  YB_CUDA_CHECK(cudaEventCreate(&a));
  YB_CUDA_CHECK(cudaEventCreate(&b));
  int rc = 0;
  for (int i = 0; i < 2 && !rc; i++) rc = once();
  if (!rc) cudaEventRecord(a, s);
  for (int i = 0; i < reps && !rc; i++) rc = once();
  if (!rc) cudaEventRecord(b, s);
  if (!rc && cudaStreamSynchronize(s) != cudaSuccess) { set_error("yb_time_op: sync failed"); rc = YB_ERR_CUDA; }
  float ms = 0.f;
  if (!rc) cudaEventElapsedTime(&ms, a, b);
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  *ms_per_launch = ms / reps;
  return rc;
}

int32_t yb_op_cost(const yb_engine* e, int32_t i, int32_t batch, double* flops, double* bytes) {
  if (!e || i < 0 || i >= (int32_t)e->ops.size() || !flops || !bytes) { set_error("yb_op_cost: bad argument"); return YB_ERR_INVALID_ARG; }
  const OpDesc& op = e->ops[i];
  auto vbytes = [&](VRef r) -> double {
    if (r.buf < 0) return 0.0;
    const BufDesc& b = e->bufs[r.buf];
    return (double)batch * b.H * b.W * r.C * e->esize;
  };
  *flops = 0;
  *bytes = vbytes(op.in) + vbytes(op.out) + vbytes(op.res) + vbytes(op.out2) + vbytes(op.out3);
  if (op.type == OP_CONV || op.type == OP_DWCONV) {
    const BufDesc& ob = e->bufs[op.out.buf];
    const double macs = (double)batch * ob.H * ob.W * op.cout * (op.cin / op.groups) * op.k * op.k;
    *flops = 2.0 * macs;
    *bytes += (double)op.cout * (op.cin / op.groups) * op.k * op.k * e->esize;
    if (op.use_tc && op.dec.mode != EPI_STORE)  // fused head tail writes fp32 straight into pred
      *bytes += vbytes(op.out) / e->esize * 4.0 - vbytes(op.out);
    if (i == 0) {  // stem reads the caller's NCHW tensor, not an engine buffer
      *bytes -= vbytes(op.in);
      *bytes += (double)batch * 3 * e->cfg.height * e->cfg.width * e->esize;
    }
    if (op.absorbed) *bytes = 0;  // moved by the fused launch of the next op
    if (op.bneck) {               // reads the block input (once, also as the shortcut) and both weight sets
      const OpDesc& pa = e->ops[i - 1];
      *bytes = vbytes(pa.in) + vbytes(op.out) + (double)(pa.cout * pa.cin + op.cout * op.cin) * 9 * e->esize;
    }
    // A folded producer launches nothing and reports no work of its own (yb_op_kind 6, like a fused Detect decode); its
    // FLOPs are the folding 1x1's, whose launch reads the producer's input and both weight sets and stores its output.
    if (op.folded) *flops = 0;
    if (op.fold) {
      const OpDesc& pa = e->ops[i - 1];
      const BufDesc& pb = e->bufs[pa.out.buf];
      *flops += 2.0 * batch * pb.H * pb.W * pa.cout * pa.cin * pa.k * pa.k;
      *bytes += vbytes(pa.in) + (double)pa.cout * pa.cin * pa.k * pa.k * e->esize - vbytes(op.in);
    }
  } else if (op.type == OP_DECODE) {
    *bytes = vbytes(op.in) + vbytes(op.cls) + vbytes(op.coef) +
             (double)batch * e->pred_c * e->bufs[op.in.buf].H * e->bufs[op.in.buf].W * 4.0;
  }
  return YB_OK;
}

/* debug: the `skip`-th tensor-core conv launch from now on records a timeline (CTA 0: MMA-issuer and first
 * epilogue warp clock64 stamps for its first 16 tiles) into dev_buf (128 x int64). */
int32_t yb_debug_timeline(long long* dev_buf, int32_t skip) {
  yb::g_tc_dbg = dev_buf;
  yb::g_tc_dbg_countdown = skip;
  return YB_OK;
}

static void copy_desc(const std::string& s, char* desc, int32_t cap) {
  if (desc && cap > 0) snprintf(desc, (size_t)cap, "%s", s.c_str());
}

// Launches a tensor-core plan (fused Bottleneck when `bn` is set) with a zeroed tile counter (or none) on the legacy
// stream and waits for it.
static int run_debug_launch(const TcConvPlan* plan, const TcBneckPlan* bn, int B, float* pred, bool tile_counter,
                            const char* who) {
  int* ctr = nullptr;
  if (tile_counter) {
    YB_CUDA_CHECK(cudaMalloc((void**)&ctr, sizeof(int)));
    YB_CUDA_CHECK(cudaMemset(ctr, 0, sizeof(int)));
  }
  int rc = bn ? tc_bneck_launch(bn, B, ctr, 0) : tc_conv_launch(plan, B, pred, ctr, 0);
  const cudaError_t ce = cudaDeviceSynchronize();
  if (!rc && ce != cudaSuccess) {
    set_error(std::string(who) + ": kernel failed: " + cudaGetErrorString(ce));
    rc = YB_ERR_CUDA;
  }
  if (ctr) cudaFree(ctr);
  return rc;
}

int32_t yb_debug_conv_f16(const void* in, int32_t plan_batch, int32_t run_batch, int32_t height, int32_t width, int32_t in_pitch,
                          int32_t in_coff, int32_t cin, const void* w, const float* bias, int32_t cout, int32_t k, int32_t stride,
                          int32_t act, const void* res, int32_t res_pitch, int32_t res_coff, void* out, int32_t out_pitch,
                          int32_t out_coff, int32_t share_sms, int32_t tile_counter, int32_t dec_mode, int32_t dec_anchors,
                          int32_t dec_channels, int32_t dec_a0, int32_t dec_ch0, int32_t dec_width, int32_t dec_pixels,
                          float dec_stride, float* pred, char* desc, int32_t desc_capacity) {
  const bool decode = dec_mode != EPI_STORE;
  if (!in || !w || !bias || (decode ? !pred : !out)) { set_error("yb_debug_conv_f16: null argument"); return YB_ERR_INVALID_ARG; }
  if (plan_batch <= 0 || run_batch <= 0 || run_batch > plan_batch || height <= 0 || width <= 0 || cin <= 0 || cout <= 0 ||
      in_coff < 0 || in_pitch < in_coff + cin || (k != 1 && k != 3) || stride <= 0 || (act != ACT_NONE && act != ACT_SILU) ||
      dec_mode < EPI_STORE || dec_mode > EPI_RAW || (!decode && (out_coff < 0 || out_pitch < out_coff + cout)) ||
      (res && (res_coff < 0 || res_pitch < res_coff + cout))) {
    set_error("yb_debug_conv_f16: bad argument (batch, extent, channel view, k, stride, act or decode mode)");
    return YB_ERR_INVALID_ARG;
  }
  ConvParams p;
  p.B = plan_batch;
  p.Cin = cin; p.Cout = cout;
  p.k = k; p.stride = stride; p.pad = k / 2;
  p.Ho = (height + 2 * p.pad - k) / stride + 1;
  p.Wo = (width + 2 * p.pad - k) / stride + 1;
  p.act = act;
  p.w = w; p.bias = bias;
  p.share_sms = share_sms ? 1 : 0;
  p.in.base = const_cast<void*>(in); p.in.H = height; p.in.W = width; p.in.pitch = in_pitch; p.in.coff = in_coff; p.in.C = cin;
  p.out.base = out; p.out.H = p.Ho; p.out.W = p.Wo; p.out.pitch = out_pitch; p.out.coff = out_coff; p.out.C = cout;
  if (res) {
    p.res.base = const_cast<void*>(res); p.res.H = p.Ho; p.res.W = p.Wo; p.res.pitch = res_pitch; p.res.coff = res_coff; p.res.C = cout;
  }
  p.dec.mode = dec_mode; p.dec.A = dec_anchors; p.dec.Ctot = dec_channels; p.dec.a0 = dec_a0; p.dec.ch0 = dec_ch0;
  p.dec.Wl = dec_width; p.dec.HW = dec_pixels; p.dec.stride = dec_stride;
  if (!tc_conv_supported(p)) {
    set_error("yb_debug_conv_f16: shape not supported by the tensor-core conv (Cin, Cout % 16, Cout <= 1024, k / stride, "
              "channel offsets and pitches % 8)");
    return YB_ERR_SHAPE;
  }
  if (!have_device("yb_debug_conv_f16")) return YB_ERR_NO_DEVICE;
  std::string err;
  TcConvPlan* plan = tc_conv_plan_create(p, &err);
  if (!plan) { set_error("yb_debug_conv_f16: " + err); return YB_ERR_SHAPE; }
  copy_desc(tc_conv_plan_describe(plan), desc, desc_capacity);
  const int rc = run_debug_launch(plan, nullptr, run_batch, pred, tile_counter != 0, "yb_debug_conv_f16");
  tc_conv_plan_destroy(plan);
  return rc;
}

int32_t yb_debug_bneck_f16(const void* x, int32_t batch, int32_t height, int32_t width, int32_t x_pitch, int32_t x_coff, int32_t cin,
                           const void* w_a, const float* bias_a, int32_t cmid, const void* w_b, const float* bias_b, int32_t cout,
                           int32_t shortcut, void* out, int32_t out_pitch, int32_t out_coff, char* desc, int32_t desc_capacity) {
  if (!x || !w_a || !bias_a || !w_b || !bias_b || !out) { set_error("yb_debug_bneck_f16: null argument"); return YB_ERR_INVALID_ARG; }
  if (batch <= 0 || height <= 0 || width <= 0 || cin <= 0 || cmid <= 0 || cout <= 0 || x_coff < 0 || x_pitch < x_coff + cin ||
      out_coff < 0 || out_pitch < out_coff + cout) {
    set_error("yb_debug_bneck_f16: bad argument (batch, extent or channel view)");
    return YB_ERR_INVALID_ARG;
  }
  // conv a writes t into a dense scratch buffer (the fused kernel never touches it: it only needs the plan), conv b reads it
  ConvParams pa;
  pa.B = batch; pa.Cin = cin; pa.Cout = cmid;
  pa.k = 3; pa.stride = 1; pa.pad = 1; pa.Ho = height; pa.Wo = width;
  pa.act = ACT_SILU; pa.w = w_a; pa.bias = bias_a;
  pa.in.base = const_cast<void*>(x); pa.in.H = height; pa.in.W = width; pa.in.pitch = x_pitch; pa.in.coff = x_coff; pa.in.C = cin;
  pa.out.H = height; pa.out.W = width; pa.out.pitch = cmid; pa.out.coff = 0; pa.out.C = cmid;
  ConvParams pb = pa;
  pb.Cin = cmid; pb.Cout = cout; pb.w = w_b; pb.bias = bias_b;
  pb.in = pa.out;
  pb.out.base = out; pb.out.pitch = out_pitch; pb.out.coff = out_coff; pb.out.C = cout;
  if (shortcut) pb.res = pa.in;
  if (!tc_conv_supported(pa) || !tc_conv_supported(pb)) {
    set_error("yb_debug_bneck_f16: shape not supported by the tensor-core conv (channels % 16, channel offsets and pitches % 8)");
    return YB_ERR_SHAPE;
  }
  if (!have_device("yb_debug_bneck_f16")) return YB_ERR_NO_DEVICE;
  void* t = nullptr;
  YB_CUDA_CHECK(cudaMalloc(&t, (size_t)batch * height * width * cmid * sizeof(__half)));
  pa.out.base = pb.in.base = t;
  std::string err;
  TcConvPlan* plan_a = tc_conv_plan_create(pa, &err);
  TcConvPlan* plan_b = plan_a ? tc_conv_plan_create(pb, &err) : nullptr;
  TcBneckPlan* bn = plan_b ? tc_bneck_plan_create(plan_a, plan_b, &err) : nullptr;
  int rc = 0;
  if (!bn) {
    set_error("yb_debug_bneck_f16: " + err);
    rc = YB_ERR_SHAPE;
  } else {
    copy_desc(tc_bneck_plan_describe(bn), desc, desc_capacity);
    rc = run_debug_launch(nullptr, bn, batch, nullptr, true, "yb_debug_bneck_f16");
  }
  tc_bneck_plan_destroy(bn);
  tc_conv_plan_destroy(plan_b);
  tc_conv_plan_destroy(plan_a);
  cudaFree(t);
  return rc;
}

int32_t yb_op_kind(const yb_engine* e, int32_t i) {
  if (!e || i < 0 || i >= (int32_t)e->ops.size()) return -1;
  const OpDesc& op = e->ops[i];
  switch (op.type) {
    case OP_CONV: return (i == 0 && e->has_stem_tc) ? 2 : (op.folded ? 6 : (op.use_tc ? 0 : 1));
    case OP_DWCONV: return 3;
    case OP_POOL: return 4;
    case OP_UPSAMPLE: return 5;
    case OP_DECODE: return 6;
    default: return 7;
  }
}

int32_t yb_launches_per_forward(const yb_engine* e) {
  if (!e) return 0;
  int n = e->has_stem_tc ? 0 : 1;  // generic path converts the input layout first
  for (const OpDesc& op : e->ops)
    if (!(op.type == OP_DECODE && op.fused) && !op.absorbed) n++;
  return n;
}

}  // extern "C"
