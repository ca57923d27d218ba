// Host side of the Bayesian SegNet operator: builds the op list from the prototxt (fusing the in-place
// BN / ReLU followers into their convolution, running everything upstream of the first sampling Dropout
// once instead of T times) and executes it on one stream.
#include "segnet.h"

#include <cuda_fp16.h>

#include <algorithm>
#include <cmath>
#include <cstring>

namespace sivo {

namespace {
int round_up(int a, int b) { return (a + b - 1) / b * b; }
float through_half(float x) { return __half2float(__float2half_rn(x)); }
template <typename T>
void upload(DevBuf& buf, const std::vector<T>& v) {
  buf.alloc(v.size() * sizeof(T));
  SIVO_CUDA(cudaMemcpy(buf.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
}
}  // namespace

int SegNet::add_tensor(const std::string& name, int n, int c, int h, int w, int cs, DType dt, bool mask) {
  auto t = std::make_unique<Tensor>();
  t->name = name;
  t->v.n = n; t->v.c = c; t->v.h = h; t->v.w = w; t->v.cs = cs; t->v.dt = dt;
  t->is_mask = mask;
  size_t bytes = mask ? static_cast<size_t>(n) * h * w * cs : t->v.bytes();
  t->buf.alloc(bytes);
  t->v.p = t->buf.p;
  tensors_.push_back(std::move(t));
  int id = static_cast<int>(tensors_.size()) - 1;
  by_name_[name] = id;
  return id;
}

TensorView split_view(TensorView v) {
  v.p = nullptr;
  v.dt = DType::F16;
  v.cs *= 2;
  return v;
}

void prepare_conv(Op& op, DType act, const float* W, const float* bias, const float* bn_scale, const float* bn_shift,
                  const TensorView& in, const TensorView& out) {
  const int K = op.k, cin = op.fold_kw ? 3 : op.cin, cout = op.cout;
  const int taps = op.fold_kw ? K : K * K;
  auto slot = [&](int t, int ci, int& tap, int& cidx) {
    // tap row kh; "channel" = window pixel * 8 + c.  The window of output pixel x starts at image pixel x - 3, tap column
    // kw reads image pixel x + kw - (K-1)/2, i.e. window pixel kw + 3 - (K-1)/2
    if (op.fold_kw) { tap = t / K; cidx = (t % K + 3 - (K - 1) / 2) * 8 + ci; }
    else { tap = t; cidx = ci; }
  };
  op.h_w_raw.assign(W, W + static_cast<size_t>(cout) * cin * K * K);
  op.h_bias.assign(op.cout_p, 0.f);
  if (bias) std::copy(bias, bias + cout, op.h_bias.begin());
  op.has_bn = bn_scale != nullptr;
  if (op.has_bn) {
    op.h_bn_scale.assign(op.cout_p, 1.f);
    op.h_bn_shift.assign(op.cout_p, 0.f);
    std::copy(bn_scale, bn_scale + cout, op.h_bn_scale.begin());
    if (bn_shift) std::copy(bn_shift, bn_shift + cout, op.h_bn_shift.begin());
  }
  if (op.split) {
    upload(op.w_tc, conv_tc_split_weights(W, cout, cin, K, op.cout_p, op.cin_p, &op.acc_scale));
    TensorView planes = split_view(in);
    op.a_split.alloc(planes.bytes());
    planes.p = op.a_split.p;
    op.tc = conv_tc_plan(op, planes, out, op.w_tc.p);
  } else if (op.use_tc) {  // [tap][cout_p][cin_p] half, K(=cin)-major rows
    std::vector<__half> wt(static_cast<size_t>(taps) * op.cout_p * op.cin_p, __float2half_rn(0.f));
    for (int co = 0; co < cout; ++co)
      for (int ci = 0; ci < cin; ++ci)
        for (int t = 0; t < K * K; ++t) {
          int tap, cidx;
          slot(t, ci, tap, cidx);
          wt[(static_cast<size_t>(tap) * op.cout_p + co) * op.cin_p + cidx] =
              __float2half_rn(W[(static_cast<size_t>(co) * cin + ci) * K * K + t]);
        }
    upload(op.w_tc, wt);
    op.tc = conv_tc_plan(op, in, out, op.w_tc.p);
  } else {  // [tap][cin_p][cout_p] float, through half for fp16 activations
    std::vector<float> ws(static_cast<size_t>(taps) * op.cin_p * op.cout_p, 0.f);
    for (int co = 0; co < cout; ++co)
      for (int ci = 0; ci < cin; ++ci)
        for (int t = 0; t < K * K; ++t) {
          float v = W[(static_cast<size_t>(co) * cin + ci) * K * K + t];
          int tap, cidx;
          slot(t, ci, tap, cidx);
          ws[(static_cast<size_t>(tap) * op.cin_p + cidx) * op.cout_p + co] = act == DType::F16 ? through_half(v) : v;
        }
    upload(op.w_simt, ws);
    upload(op.bias, op.h_bias);
    if (op.has_bn) {
      upload(op.bn_scale, op.h_bn_scale);
      upload(op.bn_shift, op.h_bn_shift);
    }
  }
}

void launch_conv(const Op& op, const TensorView& in, const TensorView& out, cudaStream_t s) {
  if (op.use_tc) {
    if (op.split) launch_split_hilo(in, op.a_split.p, s);  // the float input as [hi | lo] half planes
    conv_tc_launch(*op.tc, s);
    return;
  }
  ConvParams p;
  p.in = in;
  p.out = out;
  p.w_simt = op.w_simt.as<float>();
  p.bias = op.bias.as<float>();
  p.bn_scale = op.has_bn ? op.bn_scale.as<float>() : nullptr;
  p.bn_shift = op.has_bn ? op.bn_shift.as<float>() : nullptr;
  p.k = op.k; p.pad = op.pad; p.cin_p = op.cin_p; p.cout_p = op.cout_p;
  p.relu = op.relu; p.slope = op.slope;
  launch_conv_simt(p, s);
}

void SegNet::build(const NetSpec& net, const WeightMap& weights) {
  // consumers of each blob name, to spot the convolution feeding Softmax
  auto feeds_softmax = [&](size_t li, const std::string& top) {
    for (size_t j = li + 1; j < net.layers.size(); ++j)
      for (auto& b : net.layers[j].bottoms)
        if (b == top) return net.layers[j].type == LayerType::Softmax;
    return false;
  };
  int in_id = add_tensor(net.input_name, 1, 3, H_, W_, 4, act_);
  {
    Op op;
    op.kind = Op::Input;
    op.layer = "input";
    op.out = in_id;
    ops_.push_back(std::move(op));
  }
  auto blob_id = [&](const std::string& name) {
    auto it = by_name_.find(name);
    if (it == by_name_.end()) fail(SIVO_EFORMAT, "prototxt: blob '%s' is used before it is produced", name.c_str());
    // a fused kernel consumes this blob in registers and never writes it: a second consumer would read uninitialised memory
    if (tensors_[it->second]->elided || tensors_[it->second]->derived_from >= 0)
      fail(SIVO_EFORMAT, "prototxt: blob '%s' has more than one consumer; the fused pool / unpool / dropout / classifier paths need a "
                         "single-consumer chain (create the net with keep_blobs to run it unfused)", name.c_str());
    return it->second;
  };
  // `conv` is a 7x7 convolution that can unpool on load, reading the max-unpool the last op writes -- an Unpool, or a
  // sampling Dropout that writes its result unpooled (Basic's decoder: upsample4 .. upsample1).  The op is taken back: an
  // Unpool is dropped, a DropoutUnpool writes the pooled tensor as a plain Dropout, and `conv` expands the pooled tensor as
  // it loads its halo rows.  The unpooled tensor, three quarters zeros, is derived: never written.  The launch names stay
  // those of the scattering build: the upsample is named with the launch that produces the values it places.
  auto unpool_on_load = [&](Op& conv) {
    Op& up = ops_.back();
    int pooled;
    if (up.kind == Op::Unpool && up.out == conv.in) pooled = up.in;
    else if (up.kind == Op::DropoutUnpool && up.out2 == conv.in) pooled = up.out;
    else return;
    const Tensor& pt = *tensors_[pooled];
    const Tensor& mt = *tensors_[up.in2];
    conv_tc_set_unpool_input(*conv.tc, pt.v.p, mt.buf.as<uint8_t>(), mt.v.n, pt.v.h, pt.v.w);
    Tensor& unpooled = *tensors_[conv.in];
    unpooled.derived_from = pooled;
    unpooled.derived_mask = up.in2;
    unpooled.buf.release();
    unpooled.v.p = nullptr;
    if (up.kind == Op::Unpool) {
      const std::string name = up.layer;
      ops_.pop_back();
      if (!ops_.empty() && ops_.back().out == pooled) ops_.back().layer += "+" + name;
    } else {
      up.kind = Op::Dropout;
      tensors_[pooled]->elided = false;
      up.in2 = up.out2 = -1;
    }
  };
  int drop_idx = 0;
  bool saw_softmax = false;
  for (size_t li = 0; li < net.layers.size(); ++li) {
    const LayerSpec& ly = net.layers[li];
    if (saw_softmax) fail(SIVO_EFORMAT, "prototxt: layers after Softmax are not on the path");
    int in = blob_id(ly.bottoms[0]);
    const TensorView iv = tensors_[in]->v;
    switch (ly.type) {
      case LayerType::LRN: {
        Op op;
        op.kind = Op::LRN;
        op.layer = ly.name;
        op.in = in;
        op.out = add_tensor(ly.tops[0], iv.n, iv.c, iv.h, iv.w, iv.cs, act_);
        op.lrn_size = ly.local_size; op.lrn_alpha = ly.alpha; op.lrn_beta = ly.beta; op.lrn_k = ly.k;
        ops_.push_back(std::move(op));
        break;
      }
      case LayerType::Convolution: {
        Op op;
        op.kind = Op::Conv;
        op.layer = ly.name;
        op.in = in;
        op.k = ly.kernel; op.pad = ly.pad; op.cin = iv.c; op.cout = ly.num_output;
        op.cin_p = iv.cs;
        if (iv.cs == 4 && iv.c == 3 && act_ == DType::F16 && opt_.engine != SIVO_ENGINE_SIMT && (ly.kernel == 7 || ly.kernel == 3) &&
            ly.num_output % 64 == 0) {
          // 3-channel first layer: zero-pad to 8-channel pixels; the convolution's TMA reads overlapping 8-pixel windows of it
          // (K x 1 layer)
          Op ex;
          ex.kind = Op::Pad8;
          ex.in = in;
          ex.layer = ly.name + "/pad8";
          ex.out = add_tensor("__pad8_" + ly.name, iv.n, 8, iv.h, iv.w + 8, 8, act_);
          const size_t no = ops_.size();
          if (!opt_.keep_blobs && no >= 2 && ops_[no - 1].kind == Op::LRN && ops_[no - 1].out == in && ops_[no - 2].kind == Op::Input &&
              ops_[no - 2].out == ops_[no - 1].in && iv.n == 1) {
            // input -> LRN -> pad8 collapse into one pass (the 'data' and 'norm' blobs are not materialised)
            ex.kind = Op::InputPad8;
            ex.lrn_size = ops_[no - 1].lrn_size; ex.lrn_alpha = ops_[no - 1].lrn_alpha;
            ex.lrn_beta = ops_[no - 1].lrn_beta; ex.lrn_k = ops_[no - 1].lrn_k;
            ex.layer = "input+" + ops_[no - 1].layer + "+" + ex.layer;
            tensors_[ops_[no - 1].out]->elided = tensors_[ops_[no - 2].out]->elided = true;
            ops_.pop_back();
            ops_.pop_back();
          }
          ops_.push_back(std::move(ex));
          op.in = ops_.back().out;
          op.fold_kw = ly.kernel;
          op.cin = 64; op.cin_p = 64;
        }
        const TensorView civ = tensors_[op.in]->v;  // the tensor the convolution actually reads
        op.cout_p = round_up(op.cout, 64);
        const std::vector<Blob>* bn = nullptr;
        size_t lj = li + 1;
        for (; lj < net.layers.size(); ++lj) {  // absorb the in-place followers
          const LayerSpec& f = net.layers[lj];
          bool inplace = f.bottoms[0] == ly.tops[0] && f.tops[0] == ly.tops[0];
          if (!inplace) break;
          if (f.type == LayerType::BN && !bn && !op.relu) {
            auto it = weights.find(f.name);
            if (it == weights.end()) fail(SIVO_EFORMAT, "caffemodel has no blobs for BN layer '%s'", f.name.c_str());
            bn = &it->second;
          } else if (f.type == LayerType::ReLU && !op.relu) {
            op.relu = true;
            op.slope = f.negative_slope;
          } else {
            break;
          }
        }
        bool logits = feeds_softmax(lj - 1, ly.tops[0]);
        if (!logits && (op.cout % 8)) fail(SIVO_EFORMAT, "layer '%s': %d output channels (need a multiple of 8)", ly.name.c_str(), op.cout);
        int cs = logits ? round_up(op.cout, 16) : op.cout;
        op.out = add_tensor(ly.tops[0], iv.n, op.cout, iv.h, iv.w, cs, logits ? DType::F32 : act_);
        auto it = weights.find(ly.name);
        if (it == weights.end()) fail(SIVO_EFORMAT, "caffemodel has no blobs for layer '%s'", ly.name.c_str());
        const std::vector<Blob>& cb = it->second;
        const int wcin = op.fold_kw ? 3 : op.cin;
        if (cb.empty() || cb[0].shape.size() != 4 || cb[0].shape[0] != op.cout || cb[0].shape[1] != wcin || cb[0].shape[2] != op.k ||
            cb[0].shape[3] != op.k)
          fail(SIVO_EFORMAT, "layer '%s': weight blob shape does not match (%d,%d,%d,%d) (net.cpp:750-785 would CHECK-fail)",
               op.layer.c_str(), op.cout, wcin, op.k, op.k);
        if (cb.size() > 1 && static_cast<int>(cb[1].count()) != op.cout)
          fail(SIVO_EFORMAT, "layer '%s': bias blob size mismatch", op.layer.c_str());
        if (bn && (bn->size() < 2 || static_cast<int>((*bn)[0].count()) != op.cout || static_cast<int>((*bn)[1].count()) != op.cout))
          fail(SIVO_EFORMAT, "BN after '%s': expected scale and shift blobs of %d channels", op.layer.c_str(), op.cout);
        const float* w = cb[0].data.data();
        const float* bias = cb.size() > 1 ? cb[1].data.data() : nullptr;
        op.flops = 2.0 * iv.c * ly.kernel * ly.kernel * op.cout * iv.h * iv.w * iv.n;  // algorithmic, whatever the mapping
        flops_dedup += op.flops;
        flops_naive += op.flops / iv.n * ns_;
        if (logits && !opt_.keep_blobs && op.k == 1 && op.cin == 64 && op.cout <= 16 && !op.relu && !bn && !ops_.empty() &&
            ops_.back().kind == Op::Conv && ops_.back().use_tc && ops_.back().out == in && conv_tc_can_compose_classifier(*ops_.back().tc)) {
          // 1x1 classifier straight after a tensor-core convolution with no non-linearity between them (Basic): logits =
          // (Wc W) * x + (Wc b + bc), ONE 64 -> 16 convolution with weights composed in double and rounded to half once --
          // a quarter of the multiply-adds, the 64-channel tensor is never written or re-read, and closer to the reference's
          // fp32 arithmetic than the two layers in half (the 64-channel activation is never rounded to half;
          // tests/test_gpu_parity.py, tools/compose_classifier_study.py).  The classifier's own weights are never uploaded.
          Op& conv = ops_.back();
          conv_tc_set_composed_classifier(*conv.tc, conv, w, bias, op.cout, static_cast<float*>(tensors_[op.out]->v.p));
          // the 16-wide composed layer, warm-up rows included
          conv.flops_exec = 2.0 * conv.cin * conv.k * conv.k * 16 * iv.h * iv.w * iv.n * conv_tc_rows_ratio(*conv.tc);
          conv.layer += "*" + ly.name;  // '*': composed, not merely fused
          Op* up = ops_.size() >= 2 ? &ops_[ops_.size() - 2] : nullptr;
          if (up && tensors_[conv.in]->derived_from == up->out) {
            // the composed kernel unpools its input on load (Basic: conv_decode2 -> upsample1), and carries its name
            const size_t plus = up->layer.rfind('+');  // the unpool is the last layer named with the producer
            conv.layer = up->layer.substr(plus + 1) + "+" + conv.layer;
            up->layer.erase(plus);
          }
          conv.flops += op.flops;  // algorithmic: the reference runs both layers
          tensors_[in]->elided = true;
          li = lj - 1;
          break;
        }
        const TensorView& ov = tensors_[op.out]->v;
        // fp32 activations on the tensor-core engine: split-operand mode (three half MMAs per tap, fp32 accumulation)
        if (act_ == DType::F32 && opt_.engine != SIVO_ENGINE_SIMT && !op.fold_kw && civ.cs % 64 == 0 && civ.c == civ.cs) {
          op.split = true;
          if (!conv_tc_supported(op, split_view(civ), ov)) op.split = false;
        }
        op.use_tc = op.split || (opt_.engine != SIVO_ENGINE_SIMT && act_ == DType::F16 && conv_tc_supported(op, civ, ov));
        if (!op.use_tc && op.fold_kw)
          fail(SIVO_EINVAL, "layer '%s': window-folded first layer is not supported by the tensor-core kernel", ly.name.c_str());
        if (!op.use_tc && opt_.engine == SIVO_ENGINE_TCGEN05 && op.cin_p % 64 == 0 && (!logits || act_ == DType::F32))
          fail(SIVO_EINVAL, "layer '%s': tcgen05 engine requested but the shape is not supported", ly.name.c_str());
        prepare_conv(op, act_, w, bias, bn ? (*bn)[0].data.data() : nullptr, bn ? (*bn)[1].data.data() : nullptr, civ, ov);
        op.flops_exec = op.split ? 3.0 * op.flops : op.flops * (op.use_tc ? conv_tc_rows_ratio(*op.tc) : 1.0);
        if (!opt_.keep_blobs && op.use_tc && !ops_.empty() && conv_tc_can_unpool_input(*op.tc)) unpool_on_load(op);
        ops_.push_back(std::move(op));
        li = lj - 1;
        break;
      }
      case LayerType::ReLU:
      case LayerType::BN:
        fail(SIVO_EFORMAT, "layer '%s': %s must follow a convolution in place", ly.name.c_str(),
             ly.type == LayerType::BN ? "BN" : "ReLU");
      case LayerType::Pooling: {
        if ((iv.h | iv.w) & 1) fail(SIVO_EFORMAT, "layer '%s': odd input size %dx%d", ly.name.c_str(), iv.h, iv.w);
        if (iv.cs != iv.c) fail(SIVO_EFORMAT, "layer '%s': pooling a padded-channel tensor", ly.name.c_str());
        const int pooled = add_tensor(ly.tops[0], iv.n, iv.c, iv.h / 2, iv.w / 2, iv.cs, act_);
        const int pmask = add_tensor(ly.tops[1], iv.n, iv.c, iv.h / 2, iv.w / 2, iv.cs, act_, true);
        if (!opt_.keep_blobs && !ops_.empty() && ops_.back().kind == Op::Conv && ops_.back().use_tc && ops_.back().out == in &&
            iv.dt == DType::F16 && conv_tc_can_fuse_pool(*ops_.back().tc)) {
          // the producing tensor-core convolution pools in its epilogue: the full-resolution activations are never stored
          conv_tc_set_pool(*ops_.back().tc, tensors_[pooled]->v.p, tensors_[pmask]->buf.as<uint8_t>());
          tensors_[in]->elided = true;
          ops_.back().layer += "+" + ly.name;
          break;
        }
        Op op;
        op.kind = Op::Pool;
        op.layer = ly.name;
        op.in = in;
        op.out = pooled;
        op.out2 = pmask;
        ops_.push_back(std::move(op));
        break;
      }
      case LayerType::Upsample: {
        int m = blob_id(ly.bottoms[1]);
        const Tensor& mt = *tensors_[m];
        if (!mt.is_mask || mt.v.c != iv.c || mt.v.h != iv.h || mt.v.w != iv.w)
          fail(SIVO_EFORMAT, "layer '%s': mask blob '%s' does not match the input", ly.name.c_str(), ly.bottoms[1].c_str());
        const int up = add_tensor(ly.tops[0], iv.n, iv.c, iv.h * 2, iv.w * 2, iv.cs, act_);
        if (!opt_.keep_blobs && !ops_.empty() && ops_.back().kind == Op::Conv && ops_.back().use_tc && ops_.back().out == in &&
            iv.dt == DType::F16 && iv.cs == iv.c && conv_tc_can_fuse_unpool(*ops_.back().tc)) {
          // the producing tensor-core convolution scatters straight into the unpooled tensor (its own output blob
          // is never materialised; keep_blobs keeps the two-kernel form so tests can read it)
          conv_tc_set_unpool(*ops_.back().tc, mt.buf.as<uint8_t>(), mt.v.n, tensors_[up]->v.p);
          tensors_[in]->elided = true;
          ops_.back().layer += "+" + ly.name;
          break;
        }
        if (!opt_.keep_blobs && !ops_.empty() && ops_.back().kind == Op::Dropout && ops_.back().out == in && iv.dt == DType::F16 &&
            iv.cs == iv.c && iv.cs % 8 == 0) {
          // sampling Dropout feeding the upsample: one pass writes the unpooled tensor out2 (the dropped blob `out` is not
          // materialised)
          Op& d = ops_.back();
          tensors_[in]->elided = true;
          d.kind = Op::DropoutUnpool;
          d.in2 = m;
          d.out2 = up;
          d.layer += "+" + ly.name;
          break;
        }
        Op op;
        op.kind = Op::Unpool;
        op.layer = ly.name;
        op.in = in;
        op.in2 = m;
        op.out = up;
        ops_.push_back(std::move(op));
        break;
      }
      case LayerType::Dropout: {
        if (!ly.sample_weights_test) {  // plain test-time dropout is the identity (dropout_layer.cpp:43-45)
          by_name_[ly.tops[0]] = in;
          ++drop_idx;
          break;
        }
        if (ly.dropout_ratio != 0.5f)
          fail(SIVO_EFORMAT, "layer '%s': dropout_ratio %.3f (the keep-bit rule is specified for 0.5)", ly.name.c_str(), ly.dropout_ratio);
        if (!ops_.empty() && ops_.back().kind == Op::Conv && ops_.back().use_tc && ops_.back().out == in && iv.n == ns_ &&
            iv.dt == DType::F16 && ly.tops[0] == ly.bottoms[0]) {
          // in-place sampling Dropout right after a tensor-core convolution: applied in its epilogue registers
          conv_tc_set_dropout(*ops_.back().tc, opt_.seed, d_frame_.as<uint64_t>(), drop_idx++, 1.f / (1.f - ly.dropout_ratio), s0_);
          ops_.back().layer += "+" + ly.name;
          break;
        }
        Op op;
        op.kind = Op::Dropout;
        op.layer = ly.name;
        op.in = in;
        op.drop_layer = drop_idx++;
        op.drop_scale = 1.f / (1.f - ly.dropout_ratio);
        op.out = add_tensor(ly.tops[0], ns_, iv.c, iv.h, iv.w, iv.cs, act_);
        ops_.push_back(std::move(op));
        break;
      }
      case LayerType::Softmax: {
        if (iv.dt != DType::F32) fail(SIVO_EFORMAT, "Softmax must follow a convolution");
        n_classes_ = iv.c;
        Op op;
        op.kind = Op::Reduce;
        op.layer = ly.name;
        op.in = in;
        ops_.push_back(std::move(op));
        saw_softmax = true;
        break;
      }
    }
  }
  if (!saw_softmax) fail(SIVO_EFORMAT, "prototxt: no Softmax output layer ('prob')");
}

SegNet::SegNet(const std::string& prototxt, const std::string& caffemodel, const sivo_segnet_options& opt, int sample_begin,
               int sample_count)
    : opt_(opt) {
  // checkConfig (bayesian_segnet.cpp:80-89)
  if (prototxt.empty()) fail(SIVO_EINVAL, "model_file (.prototxt file) is empty!");
  if (caffemodel.empty()) fail(SIVO_EINVAL, "weights_file (.caffemodel file) is empty!");
  NetSpec net = parse_prototxt_file(prototxt);
  T_ = opt.T > 0 ? opt.T : net.dims[0];
  // bayesian_segnet.cpp:65-70
  if (net.dims[1] != 3) fail(SIVO_EINVAL, "Input layer must have 3 channels!");
  if (T_ <= 1) fail(SIVO_EINVAL, "Input layer must have a batch size greater than 1!");
  if (sample_count == 0) sample_count = T_;
  if (sample_begin < 0 || sample_count < 1 || sample_begin > T_ - sample_count)
    fail(SIVO_EINVAL, "sample range [%d, %d + %d) is not a non-empty part of the frame's %d samples", sample_begin, sample_begin,
         sample_count, T_);
  s0_ = sample_begin;
  ns_ = sample_count;
  H_ = net.dims[2];
  W_ = net.dims[3];
  if (H_ <= 0 || W_ <= 0) fail(SIVO_EFORMAT, "prototxt: bad input geometry %dx%d", W_, H_);
  act_ = opt.precision == SIVO_PRECISION_FP32 ? DType::F32 : DType::F16;
  WeightMap weights = read_caffemodel(caffemodel);
  device_ = opt.device;
  SIVO_CUDA(cudaSetDevice(device_));
  SIVO_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  try {  // a malformed model throws out of build(): the destructor does not run for a half-built object
    d_frame_.alloc(sizeof(FrameArgs));
    build(net, weights);
  } catch (...) {
    cudaStreamDestroy(stream_);
    stream_ = nullptr;
    throw;
  }
  const size_t hw = static_cast<size_t>(H_) * W_;
  d_bgr_.alloc(hw * 3);
  d_classes_.alloc(hw);
  d_conf_.alloc(hw * sizeof(double));
  d_ent_.alloc(hw * sizeof(double));
  h_in_.ensure(hw * 3);
  h_classes_.ensure(hw);
  h_conf_.ensure(hw * sizeof(double));
  h_ent_.ensure(hw * sizeof(double));
  SIVO_CUDA(cudaStreamSynchronize(stream_));
}

SegNet::~SegNet() {
  cudaSetDevice(device_);
  for (auto& g : graphs_) cudaGraphExecDestroy(g.exec);
  for (auto e : events_) cudaEventDestroy(e);
  if (stream_) cudaStreamDestroy(stream_);
}

void SegNet::enqueue(const uint8_t* bgr_dev, uint8_t* classes_dev, double* conf_dev, double* ent_dev, cudaStream_t s, bool timed) {
  launches = 0;
  if (timed) SIVO_CUDA(cudaEventRecord(events_[0], s));
  for (size_t i = 0; i < ops_.size(); ++i) {
    Op& op = ops_[i];
    switch (op.kind) {
      case Op::Input:
        launch_input_u8(bgr_dev, tensors_[op.out]->v, s, d_frame_.as<FrameArgs>());
        break;
      case Op::Pad8:
        launch_pad8(tensors_[op.in]->v, tensors_[op.out]->v, s);
        break;
      case Op::InputPad8:
        launch_input_lrn_pad8(bgr_dev, tensors_[op.out]->v, op.lrn_size, op.lrn_alpha, op.lrn_beta, op.lrn_k, s, d_frame_.as<FrameArgs>());
        break;
      case Op::LRN:
        launch_lrn(tensors_[op.in]->v, tensors_[op.out]->v, op.lrn_size, op.lrn_alpha, op.lrn_beta, op.lrn_k, s);
        break;
      case Op::Conv:
        if (op.split) ++launches;  // the hi / lo pass
        launch_conv(op, tensors_[op.in]->v, tensors_[op.out]->v, s);
        break;
      case Op::Pool:
        launch_pool(tensors_[op.in]->v, tensors_[op.out]->v, tensors_[op.out2]->buf.as<uint8_t>(), s);
        break;
      case Op::Unpool:
        launch_unpool(tensors_[op.in]->v, tensors_[op.in2]->buf.as<uint8_t>(), tensors_[op.in2]->v.n, tensors_[op.out]->v, s);
        break;
      case Op::Dropout: {
        DropoutParams d;
        d.seed = opt_.seed;
        d.frame_dev = d_frame_.as<uint64_t>();
        d.layer = op.drop_layer;
        d.sample0 = s0_;
        launch_dropout(tensors_[op.in]->v, tensors_[op.out]->v, d, op.drop_scale, s);
        break;
      }
      case Op::DropoutUnpool: {
        DropoutParams d;
        d.seed = opt_.seed;
        d.frame_dev = d_frame_.as<uint64_t>();
        d.layer = op.drop_layer;
        d.sample0 = s0_;
        const Tensor& mt = *tensors_[op.in2];
        launch_dropout_unpool(tensors_[op.in]->v, ns_, mt.buf.as<uint8_t>(), mt.v.n, tensors_[op.out2]->v, d, op.drop_scale, s);
        break;
      }
      case Op::Reduce: {
        const TensorView& lv = tensors_[op.in]->v;
        if (reduce_ == ReduceMode::Partial)
          launch_mc_partial(static_cast<const float*>(lv.p), lv.n, lv.c, lv.cs, lv.h * lv.w, s, d_frame_.as<FrameArgs>());
        else
          launch_mc_reduce(static_cast<const float*>(lv.p), lv.n, lv.c, lv.cs, lv.h * lv.w, classes_dev, conf_dev, ent_dev, s,
                           d_frame_.as<FrameArgs>());
        break;
      }
    }
    ++launches;
    if (timed) SIVO_CUDA(cudaEventRecord(events_[i + 1], s));
  }
}

void SegNet::semantic_keys(const sivo_keypoint* kps, int n, int max_static_class, uint8_t* kp_class, double* kp_conf, double* kp_entropy,
                           int* keep_idx, int* n_keep) {
  if (n_keep) *n_keep = 0;
  if (n < 0 || (n > 0 && !kps)) fail(SIVO_EINVAL, "semantic_keys: bad keypoint array");
  if (!last_classes_ || !last_conf_ || !last_ent_) fail(SIVO_EINVAL, "semantic_keys: no segmentation result on the device yet (or a map pointer was NULL)");
  if (n == 0) return;
  SIVO_CUDA(cudaSetDevice(device_));
  cudaStream_t s = last_stream_;  // the last run's maps may still be in flight on it
  // staging: in = int64 count | keypoints, out = int64 n_keep | conf | entropy | keep_idx | class
  const size_t in_bytes = 8 + static_cast<size_t>(n) * sizeof(sivo_keypoint), out_bytes = 8 + static_cast<size_t>(n) * 21;
  if (d_kp_.bytes < in_bytes) d_kp_.alloc(in_bytes * 2);
  if (d_kp_out_.bytes < out_bytes) d_kp_out_.alloc(out_bytes * 2);
  h_kp_.ensure(in_bytes);
  h_kp_out_.ensure(out_bytes);
  *h_kp_.as<long long>() = n;
  memcpy(h_kp_.as<long long>() + 1, kps, in_bytes - 8);
  SIVO_CUDA(cudaMemcpyAsync(d_kp_.p, h_kp_.p, in_bytes, cudaMemcpyHostToDevice, s));
  long long* o_n = d_kp_out_.as<long long>();
  double* o_conf = reinterpret_cast<double*>(o_n + 1);
  int* o_keep = reinterpret_cast<int*>(o_conf + 2 * n);
  launch_semantic_keys(reinterpret_cast<const sivo_keypoint*>(d_kp_.as<long long>() + 1), d_kp_.as<long long>(), n, last_classes_,
                       last_conf_, last_ent_, H_, W_, max_static_class, kp_class ? reinterpret_cast<uint8_t*>(o_keep + n) : nullptr,
                       kp_conf ? o_conf : nullptr, kp_entropy ? o_conf + n : nullptr, keep_idx ? o_keep : nullptr,
                       keep_idx || n_keep ? o_n : nullptr, s);
  SIVO_CUDA(cudaMemcpyAsync(h_kp_out_.p, d_kp_out_.p, out_bytes, cudaMemcpyDeviceToHost, s));
  SIVO_CUDA(cudaStreamSynchronize(s));
  const long long kept = *h_kp_out_.as<long long>();
  const double* hc = reinterpret_cast<const double*>(h_kp_out_.as<long long>() + 1);
  const int* hk = reinterpret_cast<const int*>(hc + 2 * n);
  if (kp_conf) memcpy(kp_conf, hc, static_cast<size_t>(n) * sizeof(double));
  if (kp_entropy) memcpy(kp_entropy, hc + n, static_cast<size_t>(n) * sizeof(double));
  if (kp_class) memcpy(kp_class, hk + n, n);
  if (keep_idx) memcpy(keep_idx, hk, static_cast<size_t>(kept) * sizeof(int));
  if (n_keep) *n_keep = static_cast<int>(kept);
}

void SegNet::semantic_keys_device(const sivo_keypoint* kps_dev, const long long* count_dev, int cap, int max_static_class, uint8_t* kp_class_dev,
                                  double* kp_conf_dev, double* kp_entropy_dev, int* keep_idx_dev, long long* n_keep_dev, cudaStream_t s) {
  if (!kps_dev || !count_dev || cap < 0) fail(SIVO_EINVAL, "semantic_keys: null keypoints or count, or negative capacity %d", cap);
  if (!last_classes_ || !last_conf_ || !last_ent_) fail(SIVO_EINVAL, "semantic_keys: no segmentation result on the device yet (or a map pointer was NULL)");
  SIVO_CUDA(cudaSetDevice(device_));
  if (!s) s = last_stream_;
  launch_semantic_keys(kps_dev, count_dev, cap, last_classes_, last_conf_, last_ent_, H_, W_, max_static_class, kp_class_dev, kp_conf_dev,
                       kp_entropy_dev, keep_idx_dev, n_keep_dev, s);
}

void SegNet::require_whole_frame(const char* what) const {
  if (ns_ < T_)
    fail(SIVO_EINVAL, "%s: this handle is a latency-mode shard owning samples [%d, %d) of %d; run it with "
                      "sivo_segnet_run_partial_device and turn the sum over all shards into maps with sivo_segnet_finalize_device",
         what, s0_, s0_ + ns_, T_);
}

void SegNet::run_device(const uint8_t* bgr_dev, uint8_t* classes_dev, double* conf_dev, double* ent_dev, cudaStream_t s, float* conf32_dev,
                        float* ent32_dev) {
  require_whole_frame("run_device");
  SIVO_CUDA(cudaSetDevice(device_));
  if (!s) s = stream_;
  last_classes_ = classes_dev; last_conf_ = conf_dev; last_ent_ = ent_dev; last_stream_ = s;
  FrameArgs fa{};
  fa.frame = frame_++;
  fa.bgr = bgr_dev; fa.classes = classes_dev; fa.conf = conf_dev; fa.ent = ent_dev; fa.conf32 = conf32_dev; fa.ent32 = ent32_dev;
  launch_frame(fa, s);
  run_stream_ = s;
}

void SegNet::run_partial(const uint8_t* bgr_dev, double* sum_dev, cudaStream_t s) {
  if (!bgr_dev || !sum_dev) fail(SIVO_EINVAL, "run_partial: null image or sum buffer");
  const TensorView& lv = tensors_[ops_.back().in]->v;  // the op list ends with the Reduce op (build() checks for the Softmax)
  if (lv.cs != 16 || lv.c > 16)
    fail(SIVO_EFORMAT, "run_partial: the partial sum needs the 16-channel logits layout (at most 16 classes, this net has %d)", lv.c);
  SIVO_CUDA(cudaSetDevice(device_));
  if (!s) s = stream_;
  FrameArgs fa{};
  fa.frame = frame_++;  // advances exactly as run_device does, so the shards of one frame stay in lockstep
  fa.bgr = bgr_dev; fa.sum = sum_dev;
  reduce_ = ReduceMode::Partial;
  try {
    launch_frame(fa, s);
  } catch (...) {
    reduce_ = ReduceMode::Full;
    throw;
  }
  reduce_ = ReduceMode::Full;
  run_stream_ = s;
}

const TensorView& SegNet::last_logits(const char* what) const {
  if (!run_stream_) fail(SIVO_EINVAL, "%s: the handle has not run a frame yet (the variance reads the last frame's samples)", what);
  return tensors_[ops_.back().in]->v;  // the op list ends with the Reduce op (build() checks for the Softmax)
}

void SegNet::variance_device(const uint8_t* classes_dev, double* variance_dev, cudaStream_t s) {
  if (!classes_dev || !variance_dev) fail(SIVO_EINVAL, "variance: null class map or variance buffer");
  require_whole_frame("variance");
  const TensorView& lv = last_logits("variance");
  SIVO_CUDA(cudaSetDevice(device_));
  if (!s) s = stream_;
  launch_mc_variance(static_cast<const float*>(lv.p), lv.n, lv.c, lv.cs, lv.h * lv.w, classes_dev, variance_dev, s);
}

void SegNet::variance_host(const uint8_t* classes, double* variance) {
  if (!classes || !variance) fail(SIVO_EINVAL, "computeVariance: null class map or variance buffer");
  require_whole_frame("computeVariance");
  last_logits("computeVariance");
  SIVO_CUDA(cudaSetDevice(device_));
  const size_t hw = static_cast<size_t>(H_) * W_;
  if (!d_var_classes_.p) d_var_classes_.alloc(hw);
  if (!d_var_.p) d_var_.alloc(hw * sizeof(double));
  // the caller's buffers are plain host memory: staged through the pinned buffers segmentImage uses, on the last run's stream
  cudaStream_t s = run_stream_;
  const bool pc = is_pinned_host(classes), pv = is_pinned_host(variance);
  if (!pc) memcpy(h_classes_.p, classes, hw);
  SIVO_CUDA(cudaMemcpyAsync(d_var_classes_.p, pc ? classes : h_classes_.p, hw, cudaMemcpyHostToDevice, s));
  variance_device(d_var_classes_.as<uint8_t>(), d_var_.as<double>(), s);
  SIVO_CUDA(cudaMemcpyAsync(pv ? variance : h_conf_.p, d_var_.p, hw * sizeof(double), cudaMemcpyDeviceToHost, s));
  SIVO_CUDA(cudaStreamSynchronize(s));
  if (!pv) memcpy(variance, h_conf_.p, hw * sizeof(double));
}

void SegNet::variance_partial(const uint8_t* classes_dev, double* moments_dev, cudaStream_t s) {
  if (!classes_dev || !moments_dev) fail(SIVO_EINVAL, "variance_partial: null class map or moments buffer");
  const TensorView& lv = last_logits("variance_partial");
  if (lv.cs != 16 || lv.c > 16)
    fail(SIVO_EFORMAT, "variance_partial: the moments need the 16-channel logits layout (at most 16 classes, this net has %d)", lv.c);
  SIVO_CUDA(cudaSetDevice(device_));
  if (!s) s = stream_;
  launch_mc_variance_partial(static_cast<const float*>(lv.p), lv.n, lv.c, lv.cs, lv.h * lv.w, classes_dev, moments_dev, s);
}

void SegNet::variance_finalize(const double* moments_dev, double* variance_dev, cudaStream_t s) {
  if (!moments_dev || !variance_dev) fail(SIVO_EINVAL, "variance_finalize: null moments or variance buffer");
  SIVO_CUDA(cudaSetDevice(device_));
  if (!s) s = stream_;
  launch_mc_variance_finalize(moments_dev, T_, H_ * W_, variance_dev, s);
}

void SegNet::finalize(const double* sum_dev, uint8_t* classes_dev, double* conf_dev, double* ent_dev, float* conf32_dev, float* ent32_dev,
                      cudaStream_t s) {
  if (!sum_dev) fail(SIVO_EINVAL, "finalize: null sum buffer");
  SIVO_CUDA(cudaSetDevice(device_));
  if (!s) s = stream_;
  launch_mc_finalize(sum_dev, T_, n_classes_, H_ * W_, classes_dev, conf_dev, ent_dev, conf32_dev, ent32_dev, s);
  last_classes_ = classes_dev; last_conf_ = conf_dev; last_ent_ = ent_dev; last_stream_ = s;  // semantic_keys reads these maps
}

void SegNet::launch_frame(FrameArgs fa, cudaStream_t s) {
  const uint8_t* bgr_dev = fa.bgr;
  uint8_t* classes_dev = fa.classes;
  double* conf_dev = fa.conf;
  double* ent_dev = fa.ent;
  // Everything that changes per frame -- the dropout frame counter and the caller's pointers -- goes to the device by value,
  // outside the captured graph (pipelined callers may issue the next frame before this one has started), so one graph per
  // stream serves every pointer set a caller cycles through
  launch_set_frame_args(d_frame_.as<FrameArgs>(), fa, s);
  if (profiling_) {
    while (events_.size() < ops_.size() + 1) {
      cudaEvent_t e;
      SIVO_CUDA(cudaEventCreate(&e));
      events_.push_back(e);
    }
    enqueue(bgr_dev, classes_dev, conf_dev, ent_dev, s, true);
    SIVO_CUDA(cudaEventSynchronize(events_[ops_.size()]));
    conv_ms = other_ms = reduce_ms = 0;
    op_ms.assign(ops_.size(), 0.f);
    for (size_t i = 0; i < ops_.size(); ++i) {
      float ms = 0;
      SIVO_CUDA(cudaEventElapsedTime(&ms, events_[i], events_[i + 1]));
      op_ms[i] = ms;
      if (ops_[i].kind == Op::Conv) conv_ms += ms;
      else if (ops_[i].kind == Op::Reduce) reduce_ms += ms;
      else other_ms += ms;
    }
    SIVO_CUDA(cudaEventElapsedTime(&total_ms, events_[0], events_[ops_.size()]));
    return;
  }
  // Steady state: the whole op list is one CUDA graph launch.  Everything that changes per frame lives in device
  // memory (the frame counter read by the dropout code), so the captured kernels and their arguments never change.
  bool all_tc = true;
  for (const Op& op : ops_) if (op.kind == Op::Conv && !op.use_tc) all_tc = false;  // the SIMT launcher sets attributes per launch
  if (graph_ok_ && all_tc) {
    // the graph's kernels read the image / result pointers from FrameArgs: the key is the stream (and the op-list variant) only
    cudaGraphExec_t graph_exec_ = nullptr;
    for (size_t i = 0; i < graphs_.size(); ++i)
      if (graphs_[i].stream == s && graphs_[i].reduce == reduce_) {
        std::rotate(graphs_.begin(), graphs_.begin() + i, graphs_.begin() + i + 1);  // move to front
        graph_exec_ = graphs_.front().exec;
        break;
      }
    if (!graph_exec_) {
      cudaGraph_t g = nullptr;
      cudaError_t e = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
      if (e == cudaSuccess) {
        try {
          enqueue(bgr_dev, classes_dev, conf_dev, ent_dev, s, false);
        } catch (...) {
          cudaStreamEndCapture(s, &g);
          if (g) cudaGraphDestroy(g);
          graph_ok_ = false;
          throw;
        }
        e = cudaStreamEndCapture(s, &g);
        if (e == cudaSuccess) e = cudaGraphInstantiate(&graph_exec_, g, 0);
        if (g) cudaGraphDestroy(g);
      }
      if (e != cudaSuccess) {  // fall back to plain launches for this handle
        cudaGetLastError();
        graph_ok_ = false;
        graph_exec_ = nullptr;
      } else {
        if (graphs_.size() >= kMaxGraphs) {  // a caller cycling through more streams than this re-captures the oldest
          cudaGraphExecDestroy(graphs_.back().exec);
          graphs_.pop_back();
        }
        graphs_.insert(graphs_.begin(), GraphEntry{s, reduce_, graph_exec_});
      }
    }
    if (graph_exec_) {
      SIVO_CUDA(cudaGraphLaunch(graph_exec_, s));
      return;
    }
  }
  enqueue(bgr_dev, classes_dev, conf_dev, ent_dev, s, false);
}

void SegNet::run_host(const uint8_t* bgr, int rows, int cols, size_t stride, uint8_t* classes, double* conf, double* ent) {
  require_whole_frame("segmentImage");
  if (!bgr) fail(SIVO_EINVAL, "segmentImage: null image");
  // resizeImage (bayesian_segnet.cpp:142-162): exact size passes through, larger is centre-cropped;
  // smaller yields an empty Mat in the reference (and a crash downstream) -- here an error.
  if (rows < H_ || cols < W_) fail(SIVO_EINVAL, "segmentImage: image %dx%d is smaller than the network input %dx%d", cols, rows, W_, H_);
  if (stride < static_cast<size_t>(cols) * 3) fail(SIVO_EINVAL, "segmentImage: stride smaller than a row");
  int x_tl = 0, y_tl = 0;
  if (rows != H_ || cols != W_) {
    x_tl = cols / 2 - W_ / 2;
    y_tl = rows / 2 - H_ / 2;
  }
  SIVO_CUDA(cudaSetDevice(device_));
  const size_t hw = static_cast<size_t>(H_) * W_;
  const uint8_t* src = bgr + static_cast<size_t>(y_tl) * stride + static_cast<size_t>(x_tl) * 3;
  if (is_pinned_host(bgr)) {  // crop straight out of the caller's page-locked image
    SIVO_CUDA(cudaMemcpy2DAsync(d_bgr_.p, static_cast<size_t>(W_) * 3, src, stride, static_cast<size_t>(W_) * 3, H_,
                                cudaMemcpyHostToDevice, stream_));
  } else {
    uint8_t* stage = h_in_.as<uint8_t>();
    for (int y = 0; y < H_; ++y)
      memcpy(stage + static_cast<size_t>(y) * W_ * 3, src + static_cast<size_t>(y) * stride, static_cast<size_t>(W_) * 3);
    SIVO_CUDA(cudaMemcpyAsync(d_bgr_.p, stage, hw * 3, cudaMemcpyHostToDevice, stream_));
  }
  // outputs are caller-owned plain memory (Frame copies them into itself, Frame.cc:239-241): page-locked caller
  // buffers receive the device copy directly, pageable ones go through the pinned staging buffers
  const bool pc = is_pinned_host(classes), pf = is_pinned_host(conf), pe = is_pinned_host(ent);
  uint8_t* hc = pc ? classes : h_classes_.as<uint8_t>();
  double* hf = pf ? conf : h_conf_.as<double>();
  double* he = pe ? ent : h_ent_.as<double>();
  run_device(d_bgr_.as<uint8_t>(), d_classes_.as<uint8_t>(), d_conf_.as<double>(), d_ent_.as<double>(), stream_, rec_conf32_, rec_ent32_);
  if (classes) SIVO_CUDA(cudaMemcpyAsync(hc, d_classes_.p, hw, cudaMemcpyDeviceToHost, stream_));
  if (conf) SIVO_CUDA(cudaMemcpyAsync(hf, d_conf_.p, hw * sizeof(double), cudaMemcpyDeviceToHost, stream_));
  if (ent) SIVO_CUDA(cudaMemcpyAsync(he, d_ent_.p, hw * sizeof(double), cudaMemcpyDeviceToHost, stream_));
  if (rec_classes_) SIVO_CUDA(cudaMemcpyAsync(rec_classes_, d_classes_.p, hw, cudaMemcpyDeviceToDevice, stream_));
  SIVO_CUDA(cudaStreamSynchronize(stream_));
  if (classes && !pc) memcpy(classes, h_classes_.p, hw);
  if (conf && !pf) memcpy(conf, h_conf_.p, hw * sizeof(double));
  if (ent && !pe) memcpy(ent, h_ent_.p, hw * sizeof(double));
}

void SegNet::blob(const std::string& name, float* out, size_t cap, int* n, int* c, int* h, int* w) {
  auto it = by_name_.find(name);
  if (it == by_name_.end()) fail(SIVO_EINVAL, "no blob named '%s'", name.c_str());
  Tensor& t = *tensors_[it->second];
  if (t.elided && out)
    fail(SIVO_EINVAL, "blob '%s' is not materialised in this build (a fused kernel consumes it); create the net with keep_blobs", name.c_str());
  if (n) *n = t.v.n;
  if (c) *c = t.v.c;
  if (h) *h = t.v.h;
  if (w) *w = t.v.w;
  if (!out) return;
  size_t count = static_cast<size_t>(t.v.n) * t.v.c * t.v.h * t.v.w;
  if (cap < count) fail(SIVO_ERANGE, "blob '%s' has %zu values, buffer holds %zu", name.c_str(), count, cap);
  SIVO_CUDA(cudaSetDevice(device_));
  if (t.derived_from >= 0) {  // computed from the last run's tensors it derives from, with the unpool kernel of the unfused build
    if (!t.buf.p) {
      t.buf.alloc(t.v.bytes());
      t.v.p = t.buf.p;
    }
    const Tensor& mt = *tensors_[t.derived_mask];
    launch_unpool(tensors_[t.derived_from]->v, mt.buf.as<uint8_t>(), mt.v.n, t.v, stream_);
  }
  DevBuf tmp(count * sizeof(float));
  if (t.is_mask) {
    launch_mask_to_nchw(t.buf.as<uint8_t>(), t.v.n, t.v.c, t.v.h, t.v.w, tmp.as<int>(), stream_);
    std::vector<int> hi(count);
    SIVO_CUDA(cudaMemcpyAsync(hi.data(), tmp.p, count * sizeof(int), cudaMemcpyDeviceToHost, stream_));
    SIVO_CUDA(cudaStreamSynchronize(stream_));
    for (size_t i = 0; i < count; ++i) out[i] = static_cast<float>(hi[i]);  // Caffe stores the index as float
  } else {
    launch_act_to_nchw(t.v, tmp.as<float>(), stream_);
    SIVO_CUDA(cudaMemcpyAsync(out, tmp.p, count * sizeof(float), cudaMemcpyDeviceToHost, stream_));
    SIVO_CUDA(cudaStreamSynchronize(stream_));
  }
}

}  // namespace sivo
