// net_plan.cuh -- static layer plan of the only model on the replay-step path:
// Reduced_ResNet18 (nf = 20, BasicBlock x [2,2,2,2]) and SupConResNet on top of it
// (reference models/resnet.py:14-37,69-116,140-168; utils/setup_elements.py:46-68).
//
// Parameter arena  = every learnable tensor in torch `parameters()` order and torch layout
//                    (conv OIHW, linear [out,in]) -- so a reference nn.Module can alias it.
// Packed arena     = kernel-side copies of the conv weights: forward [tap][cin][cout] and
//                    data-gradient [tap][cout][cin]; refreshed by the SGD kernel.
// BN stats arena   = per BatchNorm2d: running_mean[c] then running_var[c], module order.
#pragma once
#include <stddef.h>
#include <string.h>

#include "../../include/b200ocl.h"
#include "conv.cuh"

namespace b200ocl {

constexpr int NET_MAX_CONV = 20;
constexpr int NET_MAX_LIN = 3;
constexpr int NET_MAX_DIM = B200OCL_NET_MAX_DIM;   // largest dim_in / out_dim
constexpr float NET_BN_EPS = 1e-5f;       // nn.BatchNorm2d defaults (models/resnet.py:20)
constexpr float NET_BN_MOMENTUM = 0.1f;

struct ConvL {
  int cin, cout, ks, stride, pad;
  int hin, win, hout, wout;
  size_t w_off;     // OIHW weight in the parameter arena
  size_t pkf_off;   // packed forward weight   [ks*ks][cin][cout]
  size_t pkd_off;   // packed data-grad weight [ks*ks][cout][cin]
  size_t act_off;   // per-image offset of this conv's output inside an activation slab (floats)
  // tensor-core operand images (3x3 stride-1 convolutions only; tc_kb_f == 0 otherwise):
  //   [channel tile][K block of 32][hi | lo][NT rows x 32 fp32, 128-byte swizzle] -- byte-copyable into smem
  size_t tc_f_off, tc_d_off;  // forward / flipped data-gradient image in the packed arena
  int tc_kb_f, tc_kb_d;       // K blocks: ceil(9*cin/32), ceil(9*cout/32)
  int tc_bn_f, tc_bn_d;       // real channels per tile: min(cout,80) / min(cin,80)
  // halo-patch tensor-core kernel (conv_tcp.cu): [channel tile][32-channel slice][tap][hi | lo][NT x 32],
  // taps of the data-gradient image already flipped; tp_sl_f == 0 when the geometry is not covered
  size_t tp_f_off, tp_d_off;
  int tp_sl_f, tp_sl_d;       // slices: ceil(cin/32), ceil(cout/32)
  int tp_bn_f, tp_bn_d;       // real channels per tile: min(cout,40) / min(cin,40)
};

// padded MMA N for a channel tile of 20 / 40 / 80 channels (wgmma tiles are padded to N % 16 == 0)
inline int tc_nt(int bn) { return bn <= 20 ? 32 : (bn <= 40 ? 48 : 80); }
struct BnL {
  int c;
  size_t g_off, b_off;  // gamma / beta in the parameter arena
  size_t stat_off;      // running_mean at stat_off, running_var at stat_off + c
  size_t save_off;      // batch mean at save_off, invstd at save_off + c (train workspace)
};
struct LinL {
  int in, out;
  size_t w_off, b_off;
};
struct BlockL {
  int c1, c2, sc;  // conv indices; sc == -1 for identity shortcuts
};

struct NetPlan {
  int n_conv;
  ConvL conv[NET_MAX_CONV];
  BnL bn[NET_MAX_CONV];       // bn[i] follows conv[i]
  BlockL blk[8];
  int n_lin;
  LinL lin[NET_MAX_LIN];      // head==0: lin[0] classifier.  SupCon: lin[0] = encoder.linear (unused),
                              // 'linear' head: lin[1]; 'mlp' head: lin[1], lin[2]
  int head;                   // 0 classifier, 1 SupCon linear, 2 SupCon mlp, 3 SupCon no head
  int in_h, in_w;
  int final_h, final_w;       // layer4 spatial size
  int pooled_h, pooled_w;     // after avg_pool2d(., 4) (floor)
  int dim_in;                 // flattened encoder feature size
  int out_dim;                // logits or projection size
  size_t n_params, n_packed, n_stats, n_bn_channels;
  size_t act_per_image;       // floats per image for one full set of conv outputs
  size_t max_act_per_image;   // largest single activation per image
};

inline int conv_out(int x, int ks, int stride, int pad) { return (x + 2 * pad - ks) / stride + 1; }

// The kernels index pixels and elements of one activation tensor with 32-bit ints: N images fit when N times the
// largest activation of one image stays within INT_MAX elements.
inline bool net_batch_fits(const NetPlan& p, int N) { return (size_t)N * p.max_act_per_image <= 2147483647u; }
inline int net_max_batch(const NetPlan& p) { return (int)(2147483647u / p.max_act_per_image); }
inline int check_batch(const char* what, const NetPlan& p, int N) {
  if (net_batch_fits(p, N)) return B200OCL_OK;
  set_error("%s: N=%d images exceed the batch limit of %d for %dx%d inputs", what, N, net_max_batch(p), p.in_h, p.in_w);
  return B200OCL_EUNSUPPORTED;
}

// Packed-arena layout of one convolution (kernel-side weight copies); c.cin/cout/ks/stride/hin/win set.
inline void conv_pack_layout(ConvL& c, size_t& pk) {
  const int cin = c.cin, cout = c.cout, ks = c.ks, stride = c.stride, win = c.win;
  c.pkf_off = pk; pk += (size_t)cout * cin * ks * ks;
  c.pkd_off = pk; pk += (size_t)cout * cin * ks * ks;
  c.tc_kb_f = c.tc_kb_d = c.tp_sl_f = c.tp_sl_d = 0;
  if (ks == 3 && stride == 1 && cin % 20 == 0) {
    c.tc_bn_f = cout < 80 ? cout : 80;
    c.tc_bn_d = cin < 80 ? cin : 80;
    c.tc_kb_f = (9 * cin + 31) / 32;
    c.tc_kb_d = (9 * cout + 31) / 32;
    c.tc_f_off = pk; pk += (size_t)(cout / c.tc_bn_f) * c.tc_kb_f * 2 * tc_nt(c.tc_bn_f) * 32;
    c.tc_d_off = pk; pk += (size_t)(cin / c.tc_bn_d) * c.tc_kb_d * 2 * tc_nt(c.tc_bn_d) * 32;
  }
  // conv_tcp.cu: images for the 3x3 stride-1 convolutions on maps its strip holds (forward + data gradient)
  if (ks == 3 && stride == 1 && c.pad == 1 && cin % 20 == 0 && tcp_strip_fits(win)) {
    c.tp_bn_f = cout < 40 ? cout : 40;
    c.tp_sl_f = (cin + 31) / 32;
    c.tp_f_off = pk; pk += (size_t)(cout / c.tp_bn_f) * c.tp_sl_f * 9 * 2 * tc_nt(c.tp_bn_f) * 32;
    c.tp_bn_d = cin < 40 ? cin : 40;
    c.tp_sl_d = (cout + 31) / 32;
    c.tp_d_off = pk; pk += (size_t)(cin / c.tp_bn_d) * c.tp_sl_d * 9 * 2 * tc_nt(c.tp_bn_d) * 32;
  }
}

// Argument block of layer c's forward (dgrad = false) or data-gradient launch over N images: geometry, the weight
// images of `packed`, flip / transposed / parity_order.  The caller adds the mode and the BatchNorm fields.
inline ConvArgs conv_layer_args(const ConvL& c, int N, const float* in, const float* packed, float* out, bool dgrad) {
  ConvArgs a{};
  a.in = in;
  a.out = out;
  a.N = N;
  a.ks = c.ks; a.stride = c.stride; a.pad = c.pad;
  if (!dgrad) {
    a.w = packed + c.pkf_off;
    a.Hin = c.hin; a.Win = c.win; a.CK = c.cin;
    a.Hout = c.hout; a.Wout = c.wout; a.CN = c.cout;
    a.M = N * c.hout * c.wout;
    if (c.tc_kb_f) { a.w_tc = packed + c.tc_f_off; a.tc_kb = c.tc_kb_f; a.tc_bn = c.tc_bn_f; }
    if (c.tp_sl_f) { a.w_tp = packed + c.tp_f_off; a.tp_bn = c.tp_bn_f; a.tp_slices = c.tp_sl_f; }
    return a;
  }
  a.w = packed + c.pkd_off;
  a.Hin = c.hout; a.Win = c.wout; a.CK = c.cout;
  a.Hout = c.hin; a.Wout = c.win; a.CN = c.cin;
  a.M = N * c.hin * c.win;
  if (c.stride == 1) {
    // dx[h,w] = sum_taps dz[h+1-kh, w+1-kw] W[kh,kw]: a forward-style correlation with flipped taps
    a.flip = 1;
    if (c.tc_kb_d) { a.w_tc = packed + c.tc_d_off; a.tc_kb = c.tc_kb_d; a.tc_bn = c.tc_bn_d; }
    if (c.tp_sl_d) { a.w_tp = packed + c.tp_d_off; a.tp_bn = c.tp_bn_d; a.tp_slices = c.tp_sl_d; }
  } else {
    a.transposed = 1;
    a.parity_order = (c.stride == 2 && c.hin % 2 == 0 && c.win % 2 == 0) ? 1 : 0;
  }
  return a;
}

// Returns 0 on success, a B200OCL_E* code otherwise.
inline int build_plan(const b200ocl_net_desc& d, NetPlan& p) {
  memset(&p, 0, sizeof(p));
  if (d.nf != 20 || d.in_h < 8 || d.in_w < 8 || d.head < 0 || d.head > 3) return B200OCL_EUNSUPPORTED;
  p.head = d.head;
  p.in_h = d.in_h;
  p.in_w = d.in_w;
  size_t off = 0, pk = 0, st = 0, sv = 0, act = 0, max_act = 0;
  int nc = 0;
  auto add_conv = [&](int cin, int cout, int ks, int stride, int hin, int win) {
    ConvL& c = p.conv[nc];
    c.cin = cin; c.cout = cout; c.ks = ks; c.stride = stride; c.pad = (ks == 3) ? 1 : 0;
    c.hin = hin; c.win = win;
    c.hout = conv_out(hin, ks, stride, c.pad);
    c.wout = conv_out(win, ks, stride, c.pad);
    c.w_off = off; off += (size_t)cout * cin * ks * ks;
    conv_pack_layout(c, pk);
    c.act_off = act;
    const size_t a = (size_t)c.hout * c.wout * cout;
    act += a;
    if (a > max_act) max_act = a;
    BnL& b = p.bn[nc];
    b.c = cout;
    b.g_off = off; off += cout;
    b.b_off = off; off += cout;
    b.stat_off = st; st += 2 * (size_t)cout;
    b.save_off = sv; sv += 2 * (size_t)cout;
    return nc++;
  };
  int h = d.in_h, w = d.in_w;
  add_conv(3, d.nf, 3, 1, h, w);  // stem (resnet.py:73-74)
  int cin = d.nf, bi = 0;
  for (int li = 0; li < 4; ++li) {
    const int cout = d.nf << li;
    for (int b = 0; b < 2; ++b, ++bi) {
      const int stride = (b == 0 && li > 0) ? 2 : 1;
      BlockL& B = p.blk[bi];
      B.c1 = add_conv(cin, cout, 3, stride, h, w);
      const int ho = p.conv[B.c1].hout, wo = p.conv[B.c1].wout;
      B.c2 = add_conv(cout, cout, 3, 1, ho, wo);
      B.sc = (stride != 1 || cin != cout) ? add_conv(cin, cout, 1, stride, h, w) : -1;
      cin = cout; h = ho; w = wo;
    }
  }
  p.n_conv = nc;
  p.final_h = h; p.final_w = w;
  p.pooled_h = h / 4; p.pooled_w = w / 4;
  if (p.pooled_h < 1 || p.pooled_w < 1) return B200OCL_EUNSUPPORTED;
  p.dim_in = cin * p.pooled_h * p.pooled_w;
  auto add_lin = [&](int in, int out) {
    LinL& l = p.lin[p.n_lin++];
    l.in = in; l.out = out;
    l.w_off = off; off += (size_t)in * out;
    l.b_off = off; off += out;
  };
  if (d.head == 0) {
    add_lin(p.dim_in, d.num_classes);
    p.out_dim = d.num_classes;
  } else {
    add_lin(d.nf * 8, 100);  // SupConResNet.encoder = Reduced_ResNet18(100): present, never used (resnet.py:144)
    if (d.head == 1) {
      add_lin(p.dim_in, d.feat_dim);
      p.out_dim = d.feat_dim;
    } else if (d.head == 2) {
      add_lin(p.dim_in, p.dim_in);
      add_lin(p.dim_in, d.feat_dim);
      p.out_dim = d.feat_dim;
    } else {
      p.out_dim = p.dim_in;
    }
  }
  // the linear forward keeps a row of at most NET_MAX_DIM weights in registers, the NCM class means a feature of as many
  // dimensions (dim_in 2560 at 128x128)
  if (p.dim_in > NET_MAX_DIM || p.out_dim > NET_MAX_DIM) return B200OCL_EUNSUPPORTED;
  p.n_params = off;
  p.n_packed = pk;
  p.n_stats = st;
  p.n_bn_channels = sv / 2;
  p.act_per_image = act;
  p.max_act_per_image = max_act;
  return B200OCL_OK;
}

// net_fwd.cu: the plan of a network state whose pointers and description check out (otherwise the error is set and
// returned), and the refresh of the packed arena from a parameter arena.
int check_state(const b200ocl_net_desc* desc, const b200ocl_net_state* st, NetPlan& p);
int launch_pack(const NetPlan& p, const float* params, float* packed, cudaStream_t stream);

}  // namespace b200ocl
