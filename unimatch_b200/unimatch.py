"""Drop-in `UniMatch(nn.Module)`: the reference's constructor, `forward()` signature, `state_dict` layout and
`{'flow_preds': [...]}` output (reference `unimatch/unimatch.py:17-26, :95-111, :365-367`), with the matching
path executed by libunimatch_sm100 (hand-written sm_90a kernels) instead of eager PyTorch ops.

Host side = plain PyTorch orchestration:
  * parameters live in a module tree generated from `spec.param_spec` (same keys/shapes as the reference);
  * activations are channel-last end to end: feature maps are token matrices [N, L=h*w, 128] (N = 2 x pairs:
    all first views, then all second views), flow-like maps are [B, h, w, F];
  * `concat1` of the reference transformer (transformer.py:271-286) is never materialised: the cross-attention
    kernel reads keys/values of the partner stream (n + N/2) mod N;
  * loop-invariant / dead work of the refinement loop is hoisted (`refine_proj`, unimatch.py:315-320) or skipped
    (mask head on non-final iterations, unimatch.py:333,351) -- results are unchanged.
Every Linear layer, the CNN backbone, the update-block convolutions, the `upsampler` head and the propagation
projections run on the library's wgmma implicit-GEMM kernel (`um_conv2d_tc`, fp32-faithful split-fp16 operands);
attention / correlation on the wgmma attention kernel.  There is no cuDNN / cuBLAS call on the path and no
alternative backend in this module.

The forward pass is a sequence of `_stage_*` methods (encoder, position + warp, transformer, correlation,
propagation, refinement iteration, upsampling) so that the parity tests can teacher-force every stage with the
oracle's intermediate tensors at the BASELINE shapes (tests/test_stages_gpu.py).

Inference only (the reference's callers use eval()/no_grad, evaluate_flow.py:19,33); `train()` mode raises.
"""
import math
from collections import namedtuple
from contextlib import contextmanager

import torch
import torch.nn as nn

from . import ops
from .spec import param_spec

_OPS = torch.ops.unimatch_sm100


class _Layer(namedtuple("_Layer", "weights bias kh kw pad_h pad_w stride cout bn mode act gamma beta k")):
    """A tensor-core convolution / Linear layer for um_conv2d_tc: weight planes (`ops.prep_conv_weight`, cout padded to a
    multiple of the output-channel tile bn), 'same' zero padding, default stride, epilogue (mode, act, LayerNorm gamma / beta)
    and k = cin * kh * kw, the real (unpadded) reduction length: 2 k FLOPs per output value."""
    __slots__ = ()

    def out_hw(self, h, w, stride):
        return (h + 2 * self.pad_h - self.kh) // stride + 1, (w + 2 * self.pad_w - self.kw) // stride + 1


def _layer(w, cin_splits, bn, bias=None, act=ops.ACT_NONE, mode=ops.CONV_LINEAR, gamma=None, beta=None, stride=1):
    """_Layer of the fp32 weight [cout, cin, kh, kw] or [cout, cin] (Linear), input channels from sources of cin_splits."""
    if w.dim() == 2:
        w = w[:, :, None, None]
    cout, cin, kh, kw = w.shape
    return _Layer(ops.prep_conv_weight(w, cin_splits, (cout + bn - 1) // bn * bn), bias, kh, kw, kh // 2, kw // 2, stride,
                  cout, bn, mode, act, gamma, beta, cin * kh * kw)


class _Node(nn.Module):
    """Parameter container; gives the flat spec table the reference's dotted state_dict names."""


def _attach(root, key, param):
    parts = key.split(".")
    node = root
    for name in parts[:-1]:
        if name not in node._modules:
            node.add_module(name, _Node())
        node = node._modules[name]
    node.register_parameter(parts[-1], param)


def _sine_table(wh, ww):
    """PositionEmbeddingSine on a wh x ww window (position.py:26-45) as a [wh, ww, 128] table:
    channels 0..63 encode y, 64..127 encode x; sin on even, cos on odd feature indices."""
    y = torch.arange(1, wh + 1, dtype=torch.float32)
    x = torch.arange(1, ww + 1, dtype=torch.float32)
    y = y / (float(wh) + 1e-6) * (2 * math.pi)
    x = x / (float(ww) + 1e-6) * (2 * math.pi)
    n = torch.arange(64, dtype=torch.float32)
    dim_t = 10000 ** (2 * torch.div(n, 2, rounding_mode="floor") / 64)
    even = (torch.arange(64) % 2 == 0)

    def enc(v):
        a = v[:, None] / dim_t
        return torch.where(even, a.sin(), a.cos())

    ey, ex = enc(y), enc(x)
    return torch.cat((ey[:, None, :].expand(wh, ww, 64), ex[None, :, :].expand(wh, ww, 64)), dim=2).contiguous()


def _ceil16(n):
    return (n + 15) // 16 * 16


class UniMatch(nn.Module):
    def __init__(self, num_scales=1, feature_channels=128, upsample_factor=8, num_head=1, ffn_dim_expansion=4,
                 num_transformer_layers=6, reg_refine=False, task="flow"):
        super().__init__()
        if feature_channels != 128:
            raise ValueError("libunimatch_sm100 is built for feature_channels=128 (main_flow.py:73)")
        if num_head != 1:
            raise NotImplementedError("multi-head attention is not implemented (as in transformer.py:63-66)")
        self.feature_channels = feature_channels
        self.num_scales = num_scales
        self.upsample_factor = upsample_factor
        self.reg_refine = reg_refine
        self.num_transformer_layers = num_transformer_layers
        self.task_built = task
        self._spec = param_spec(num_scales, feature_channels, upsample_factor, num_head, ffn_dim_expansion,
                                num_transformer_layers, reg_refine, task)
        for key, shape in self._spec.items():
            _attach(self, key, nn.Parameter(self._init_tensor(key, shape)))
        self._prep_key = None
        self._prep = None
        self._tables = {}
        self._cands = {}             # depth candidate vectors, per (min, max, n, device)
        self._attn_ws = {}           # window-major attention operand planes, cached per (device, streams, geometry)
        self._pad_ws = {}            # zero-padded plane buffers, cached per (use, shape)
        self.training = False        # inference-only module: starts (and stays) in eval mode
        self.kernel_timer = None     # bench hook: dict -> CUDA-event pairs around launch groups

    @staticmethod
    def _init_tensor(key, shape):
        # same families as the reference initialisers (backbone.py:88-95, transformer.py:222-224, attention.py:180-182)
        t = torch.empty(shape)
        if len(shape) == 4:
            nn.init.kaiming_normal_(t, mode="fan_out", nonlinearity="relu")
        elif len(shape) == 2:
            nn.init.xavier_uniform_(t)
        elif ".norm" in key:
            t.fill_(1.0 if key.endswith("weight") else 0.0)
        else:
            t.uniform_(-0.05, 0.05)
        return t

    def train(self, mode=True):
        if mode:
            raise NotImplementedError("unimatch_b200.UniMatch is inference-only (use .eval(); training stays on the reference)")
        return super().train(False)

    # ------------------------------------------------------------------------------------------ weights
    def _prepared(self):
        """`_Layer`s of every tensor-core layer, rebuilt when a parameter changes."""
        params = dict(self.named_parameters())
        key = (tuple((p._version, p.data_ptr()) for p in params.values()),)
        if self._prep_key == key:
            return self._prep
        w = {k: v.detach() for k, v in params.items()}
        LN = ops.CONV_LN
        P = {"raw": w, "blocks": []}
        for i in range(self.num_transformer_layers):
            sk, ck = "transformer.layers.%d.self_attn." % i, "transformer.layers.%d.cross_attn_ffn." % i
            w_in = torch.cat([w[sk + "q_proj.weight"], w[sk + "k_proj.weight"], w[sk + "v_proj.weight"],
                              w[ck + "k_proj.weight"], w[ck + "v_proj.weight"]], dim=0)        # [640, 128]
            hid = w[ck + "mlp.0.weight"].shape[0]
            P["blocks"].append(dict(
                tc_in=_layer(w_in, [128], 128),
                tc_m_s=_layer(w[sk + "merge.weight"], [128], 128, mode=LN, gamma=w[sk + "norm1.weight"], beta=w[sk + "norm1.bias"]),
                tc_q_c=_layer(w[ck + "q_proj.weight"], [128], 128),
                tc_m_c=_layer(w[ck + "merge.weight"], [128], 128, mode=LN, gamma=w[ck + "norm1.weight"], beta=w[ck + "norm1.bias"]),
                # the two-launch FFN; the fused FFN kernel reads the same weight planes, gamma and beta
                tc_w1=_layer(w[ck + "mlp.0.weight"], [128, 128], 256, act=ops.ACT_GELU),
                tc_w2=_layer(w[ck + "mlp.2.weight"], [hid], 128, mode=LN, gamma=w[ck + "norm2.weight"], beta=w[ck + "norm2.bias"])))
        P["tcb"] = self._prepare_backbone(w, self.num_scales)
        # SelfAttnPropagation projections (attention.py:177-178, :204-205, :227-232)
        qw, qb = w["feature_flow_attn.q_proj.weight"], w["feature_flow_attn.q_proj.bias"]
        kw, kb = w["feature_flow_attn.k_proj.weight"], w["feature_flow_attn.k_proj.bias"]
        P["prop_q"] = _layer(qw, [128], 128, qb.contiguous())
        P["prop_k"] = _layer(kw, [128], 128, kb.contiguous())
        P["prop_qk"] = _layer(torch.cat([qw, kw], 0), [128], 128, torch.cat([qb, kb]).contiguous())
        if self.reg_refine:
            P["tc"] = self._prepare_refine(w)
        if "upsampler.0.weight" in w:                                           # unimatch.py:47-52
            w0 = w["upsampler.0.weight"]                                        # [256, 2 + 128, 3, 3], input = cat(flow, feature)
            w0 = torch.cat([w0[:, 2:], w0[:, :2]], dim=1)                       # our planes hold [feature | flow]
            w2 = w["upsampler.2.weight"]
            P["up"] = dict(c0=_layer(w0, [130], 128, w["upsampler.0.bias"], act=ops.ACT_RELU),
                           c2=_layer(w2, [256], 192 if w2.shape[0] % 192 == 0 else 64, w["upsampler.2.bias"]))
        self._prep_key, self._prep = key, P
        return P

    @staticmethod
    def _prepare_backbone(w, num_scales):
        """`_Layer`s of the CNN encoder convolutions (backbone.py:49-86); layer2 and layer3 (one scale) start at stride 2."""
        first_stride = {"layer2": 2, "layer3": 2 if num_scales == 1 else 1}
        T = {}
        for key, wt in w.items():
            if not key.startswith("backbone.") or not key.endswith(".weight") or key == "backbone.conv1.weight":
                continue
            name = key[:-7]
            part = name.split(".")                  # backbone.layer<i>.<block>.conv1 | .conv2 | .downsample.0
            stride = first_stride.get(part[1], 1) if part[2:3] == ["0"] and part[3] in ("conv1", "downsample") else 1
            bn = 128 if wt.shape[0] > 64 else 64    # 96 channels: one padded 128-wide tile beats two 64-wide (A is read once)
            T[name] = _layer(wt, [wt.shape[1]], bn, w.get(name + ".bias"), stride=stride)
        return T

    @staticmethod
    def _prepare_refine(w):
        """`_Layer`s of the refinement: refine_proj and the update block (reg_refine.py:6-119)."""
        R = ops.ACT_RELU
        T = {}
        pw, pb = w["refine_proj.weight"], w["refine_proj.bias"]
        T["proj_net"] = _layer(pw[:128], [128], 128, pb[:128].contiguous(), act=ops.ACT_TANH)
        T["proj_inp"] = _layer(pw[128:], [128], 128, pb[128:].contiguous(), act=R)
        e = "refine.encoder."
        T["convc1"] = _layer(w[e + "convc1.weight"], [81], 256, w[e + "convc1.bias"], act=R)
        T["convc2"] = _layer(w[e + "convc2.weight"], [256], 96, w[e + "convc2.bias"], act=R)
        T["convf2"] = _layer(w[e + "convf2.weight"], [128], 64, w[e + "convf2.bias"], act=R)
        T["conv"] = _layer(w[e + "conv.weight"], [256], 128, w[e + "conv.bias"], act=R)
        # SepConvGRU (reg_refine.py:22-52) over hx = cat[h, inp, motion | flow] (128 + 128 + 128 channels).  `inp` is the same in
        # every refinement iteration and so is `h` of the first half (net is not carried between iterations, unimatch.py:315-333):
        # their share of each convolution is computed ONCE per forward ("_fix" weights -> a fp32 tensor the per-iteration
        # convolution adds to its accumulator) and only the channels that changed are convolved per iteration ("_var").
        g = "refine.gru.conv"
        Z, Q = ops.CONV_GRU_ZR, ops.CONV_GRU_Q
        for sfx in ("1", "2"):
            wzr = torch.cat([w[g + "z%s.weight" % sfx], w[g + "r%s.weight" % sfx]], 0)           # [256, 384, kh, kw]
            bzr = torch.cat([w[g + "z%s.bias" % sfx], w[g + "r%s.bias" % sfx]])
            wq, bq = w[g + "q%s.weight" % sfx], w[g + "q%s.bias" % sfx]                           # [128, 384, kh, kw]
            if sfx == "1":
                T["zr1_fix"] = _layer(wzr[:, :256], [128, 128], 128, bzr)                          # h0 | inp
                T["zr1_var"] = _layer(wzr[:, 256:], [128], 128, mode=Z)                            # motion | flow
            else:
                T["zr2_fix"] = _layer(wzr[:, 128:256], [128], 128, bzr)                            # inp
                T["zr2_var"] = _layer(torch.cat([wzr[:, :128], wzr[:, 256:]], 1), [128, 128], 128, mode=Z)  # h1 | motion
            T["q%s_fix" % sfx] = _layer(wq[:, 128:256], [128], 128, bq)                            # inp
            T["q%s_var" % sfx] = _layer(torch.cat([wq[:, :128], wq[:, 256:]], 1), [128, 128], 128, mode=Q)  # r*h | motion
        T["fh1"] = _layer(w["refine.flow_head.conv1.weight"], [128], 128, w["refine.flow_head.conv1.bias"], act=R)
        T["fh2"] = _layer(w["refine.flow_head.conv2.weight"], [256], 16, w["refine.flow_head.conv2.bias"])
        if "refine.mask.0.weight" in w:
            T["mask0"] = _layer(w["refine.mask.0.weight"], [128], 128, w["refine.mask.0.bias"], act=R)
            T["mask2"] = _layer(w["refine.mask.2.weight"], [256], 64, w["refine.mask.2.bias"])
        return T

    def _pos_table(self, wh, ww, device):
        k = (wh, ww, str(device))
        if k not in self._tables:
            self._tables[k] = _sine_table(wh, ww).to(device)
        return self._tables[k]

    # ------------------------------------------------------------------------------------------ timers (bench hooks)
    @contextmanager
    def _section(self, name):
        t = self.kernel_timer
        if t is None:
            yield
            return
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        yield
        e1.record()
        t.setdefault("_events", []).append(("sec:" + name, e0, e1, 0.0))

    def _timed(self, tag, flops, fn, *a):
        """bench hook: CUDA events around one launch group + its algorithmic FLOPs (no effect without a timer)."""
        t = self.kernel_timer
        if t is None:
            return fn(*a)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn(*a)
        e1.record()
        t.setdefault("_events", []).append((tag, e0, e1, flops))
        return out

    def _conv(self, layer, src0, src1=None, stride=None, rows=0, out_f32=None, off_f32=0, out_split=None, off_split=0,
              aux0=None, aux1=None, **kw):
        """um_conv2d_tc of the `_Layer` on src0 (| src1); the other arguments are those of `ops.conv2d_tc`, and `stride`
        overrides the layer's.  Under the bench timer also records 2 x output pixels x cout x k as algorithmic FLOPs."""
        stride = layer.stride if stride is None else stride

        def launch():
            _OPS.conv2d_tc(src0=src0, src1=src1, weights=layer.weights, bias=layer.bias, kh=layer.kh, kw=layer.kw,
                           pad_h=layer.pad_h, pad_w=layer.pad_w, cout=layer.cout, bn=layer.bn, mode=layer.mode, act=layer.act,
                           out_f32=out_f32, off_f32=off_f32, out_split=out_split, off_split=off_split, aux0=aux0, aux1=aux1,
                           gamma=layer.gamma, beta=layer.beta, stride=stride, rows=rows, **kw)
        if self.kernel_timer is None:
            return launch()
        pix = rows or src0.shape[1] * math.prod(layer.out_hw(src0.shape[2], src0.shape[3], stride))
        return self._timed("conv", 2.0 * pix * layer.cout * layer.k, launch)

    # ------------------------------------------------------------------------------------------ backbone
    def _stage_backbone(self, P, img0, img1, normalise):
        """CNNEncoder (backbone.py:104-133) with every 3x3 / 1x1 convolution on the wgmma implicit-GEMM kernel and
        InstanceNorm + ReLU + residual as fused bandwidth passes that emit the next convolution's fp16 planes.
        The 7x7 stem (3 input channels) is the direct fp32 kernel `um_conv7x7_small` with `normalize_img` folded into its load.
        Returns the feature maps low -> high resolution, each [2B, h, w, 128] (first views, then second views)."""
        T = P["tcb"]
        dev = img0.device
        nb = img0.shape[0] + (img1.shape[0] if img1 is not None else 0)
        C, IS, IA = self._conv, _OPS.instance_norm_stats, _OPS.instance_norm_apply
        pad64 = lambda c: (c + 63) // 64 * 64

        nplanes = [0]

        def planes(h, w, c):
            cp = pad64(c)
            if cp == c:
                return torch.empty((2, nb, h, w, cp), device=dev, dtype=torch.float16)
            nplanes[0] += 1                                  # distinct live buffers of one forward get distinct cache slots
            return self._zero_padded("backbone%d" % nplanes[0], (2, nb, h, w, cp), dev)

        def conv(src_s, name, h, w, stride=None):
            layer = T[name]
            out = torch.empty((nb, *layer.out_hw(h, w, layer.stride if stride is None else stride), layer.cout), device=dev)
            C(layer, src_s, out_f32=out, stride=stride)
            return out

        hh, ww = img0.shape[2], img0.shape[3]
        a = torch.empty((nb, (hh - 1) // 2 + 1, (ww - 1) // 2 + 1, 64), device=dev)
        if normalise:                                        # normalize_img (utils.py:23-31) folded into the stem's load
            mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
            scale = [1.0 / (255.0 * s_) for s_ in std]
            shift = [-m_ / s_ for m_, s_ in zip(mean, std)]
        else:
            scale = shift = None
        _OPS.conv7x7_small(img0, img1, True, P["raw"]["backbone.conv1.weight"], None, 2, False, scale, shift, a, None)
        h, w = a.shape[1], a.shape[2]
        cur_f = torch.empty((nb, h, w, 64), device=dev)
        cur_s = planes(h, w, 64)
        IA(a, IS(a), True, None, None, False, cur_f, cur_s, 0)
        for li in (1, 2, 3):
            for bi in range(2):
                pf = "backbone.layer%d.%d." % (li, bi)
                a1 = conv(cur_s, pf + "conv1", h, w)
                _, ho, wo, cout = a1.shape
                t_s = planes(ho, wo, cout)
                IA(a1, IS(a1), True, None, None, False, None, t_s, 0)
                a2 = conv(t_s, pf + "conv2", ho, wo)
                if (pf + "downsample.0") in T:
                    res = conv(cur_s, pf + "downsample.0", h, w)
                    st_res = IS(res)
                else:
                    res, st_res = cur_f, None
                out_f = torch.empty((nb, ho, wo, cout), device=dev)
                out_s = planes(ho, wo, cout)
                IA(a2, IS(a2), True, res, st_res, True, out_f, out_s, 0)
                cur_f, cur_s, h, w = out_f, out_s, ho, wo
        x6 = torch.empty((nb, h, w, 128), device=dev)
        x6_s = planes(h, w, 128) if self.num_scales > 1 else None
        C(T["backbone.conv2"], cur_s, out_f32=x6, out_split=x6_s)
        if self.num_scales == 1:
            return [x6]
        strides = (1, 2, 4, 8)[:self.num_scales]                               # trident_conv.py:64-70
        feats = [conv(x6_s, "backbone.trident_conv", h, w, stride=s) for s in strides]
        return feats[::-1]

    # ------------------------------------------------------------------------------------------ transformer
    @staticmethod
    def _attn_plan(attn_type, splits, h, w, layer_idx):
        """(self geometry, cross geometry) as (kh, kw, sh, sw, mask) -- the dispatch of transformer.py:62-135,
        decided statically per call site instead of the reference's data-dependent `is_self_attn` sync (:55)."""
        shift = ("swin" in attn_type) and splits > 1 and layer_idx % 2 == 1
        full2d = (1, 1, 0, 0, ops.MASK_NONE)
        if splits > 1:
            wh, ww = h // splits, w // splits
            swin2d = (splits, splits, wh // 2 if shift else 0, ww // 2 if shift else 0,
                      ops.MASK_SWIN if shift else ops.MASK_NONE)
            swin1d = (h, splits, 0, ww // 2 if shift else 0, ops.MASK_SWIN if shift else ops.MASK_NONE)
        full1d = (h, 1, 0, 0, ops.MASK_NONE)
        if attn_type == "swin" and splits > 1:
            return swin2d, swin2d
        if attn_type == "self_swin2d_cross_1d":
            return (swin2d if splits > 1 else full2d), full1d
        if attn_type == "self_swin2d_cross_swin1d":
            return (swin2d if splits > 1 else full2d), (swin1d if splits > 1 else full1d)
        return full2d, full2d

    def _zero_padded(self, tag, shape, dev):
        """fp16 plane buffer whose padding channels must read as zero (e.g. 96 -> 128, 81 -> 128 channels): zero-filled once
        and cached per (use, shape) -- the kernels only ever write the real channels, so the padding stays zero and the
        per-forward fills (6 x 200 MB at the bench shape) disappear."""
        key = (tag, tuple(shape), str(dev))
        buf = self._pad_ws.get(key)
        if buf is None:
            if len(self._pad_ws) >= 24:
                self._pad_ws.clear()
            buf = torch.zeros(shape, device=dev, dtype=torch.float16)
            self._pad_ws[key] = buf
        return buf

    def _attn_planes(self, dev, n, h, w, kh, kw, lp):
        """Window-major operand planes [6 operands: q k v (self) | k v (cross) | q (cross)][2][n][windows][lp][128], zeroed once:
        the producers only ever write rows < lw of a window, so the padding rows stay zero across layers and calls."""
        key = (str(dev), n, h, w, kh, kw, lp)
        buf = self._attn_ws.get(key)
        if buf is None:
            if len(self._attn_ws) >= 4:                   # a handful of (scale, batch) shapes; do not hoard HBM beyond that
                self._attn_ws.clear()
            buf = torch.zeros((6, 2, n, kh * kw, lp, 128), device=dev, dtype=torch.float16)
            self._attn_ws[key] = buf
        return buf

    def cached_buffers(self):
        """The device buffers this module keeps between calls: the window-major attention operand planes and the zero-padded
        plane buffers.  Each cache drops its entries once enough other shapes come along, and the caching allocator then hands
        that memory to the next allocation.  A CUDA graph captured around a forward holds their raw addresses, so whoever
        replays it must hold these tensors, taken just after the capture, for as long as the graph lives."""
        return list(self._attn_ws.values()) + list(self._pad_ws.values())

    def _stage_transformer(self, P, x, h, w, attn_type, splits, tag="s0"):
        """FeatureTransformer.forward (transformer.py:226-294) on tokens x [N, L, 128], N = 2 x pairs.  Every Linear is a
        wgmma GEMM over token rows (activations travel as fp16 (hi, lo) planes [2, rows, C] between GEMMs); LayerNorm
        (+residual) / GELU are GEMM epilogues; `cat([source, message])` of the FFN (transformer.py:141) is a second GEMM
        source.  Where the window geometry runs on the tensor-core attention kernel, the q|k|v projections write the
        kernel's window-major operand planes directly (no fp32 q/k/v, no split pass) and the attention writes the merge
        layer's operand planes.  Returns (tokens fp32 [N, L, 128], their fp16 planes [2, rows_padded, 128])."""
        n, l, c = x.shape
        half = n // 2
        rows = n * l
        rp = _ceil16(rows)
        dev = x.device
        G = self._conv
        mk = torch.empty if rp == rows else torch.zeros
        planes = lambda cp: mk((2, rp, cp), device=dev, dtype=torch.float16)
        f32 = lambda cols: mk((rp, cols), device=dev)
        tok = lambda t, c0, c1: t[:rows].view(n, l, t.shape[-1])[:, :, c0:c1]
        hid = P["blocks"][0]["tc_w1"].cout
        x_f, xo_f, x1_f = f32(c), f32(c), f32(c)
        x_s, xo_s, x1_s, msg_s, m_s = planes(c), planes(c), planes(c), planes(c), planes(c)
        # FFN: one fused kernel (the 1024-wide hidden activation stays in registers) when the rows are a multiple of 256;
        # else two GEMM launches around hidden planes in HBM
        fused_ffn = ops.ffn_tc_supported(rp)
        hid_s = None if fused_ffn else planes(hid)
        x_f[:rows] = x.reshape(rows, c)
        _OPS.split_planes(x_f, x_s, 0)
        y = q_f = None
        for i, blk in enumerate(P["blocks"]):
            geo_s, geo_c = self._attn_plan(attn_type, splits, h, w, i)
            gs, gc = (h, w) + geo_s, (h, w) + geo_c
            lp_s = ops.attention_planes_lp(*gs)
            lp_c = ops.attention_planes_lp(*gc) if geo_c == geo_s else 0      # cross planes only when they share the buffers
            ws = self._attn_planes(dev, n, h, w, geo_s[0], geo_s[1], lp_s) if lp_s else None
            # ---- q_s | k_s | v_s | k_c | v_c = x W_in^T
            win_c1 = 640 if lp_c else (384 if lp_s else 0)
            if win_c1 < 640 and y is None:
                y = f32(5 * c)
            G(blk["tc_in"], x_s, rows=rp, out_f32=y if win_c1 < 640 else None, win_dst=ws[:win_c1 // 128] if win_c1 else None,
              win_geom=gs if win_c1 else None, win_c1=win_c1, win_streams=n)
            # ---- self-attention -> merge + LayerNorm + residual (transformer.py:137-144, no FFN: :157-161)
            fl_s, fl_c = (4.0 * (l // (g[0] * g[1])) * l * 128 * n for g in (geo_s, geo_c))   # 4 Lw^2 C per window per stream
            if lp_s:
                self._timed("attn:" + tag, fl_s, _OPS.window_attention_planes, ws[0], ws[1], ws[2], n, 0, *gs, None, msg_s)
            else:
                msg = self._timed("attn_simt:" + tag, fl_s, _OPS.window_attention, tok(y, 0, 128), tok(y, 128, 256), tok(y, 256, 384), 0, *gs)
                _OPS.split_planes(msg.view(rows, c), msg_s, 0)
            G(blk["tc_m_s"], msg_s, rows=rp, out_f32=x1_f, out_split=x1_s, aux0=x_f)
            # ---- cross-attention: q from the updated stream, k / v from the partner stream's projections
            if lp_c:
                G(blk["tc_q_c"], x1_s, rows=rp, win_dst=ws[5:6], win_geom=gc, win_c1=128, win_streams=n)
                self._timed("attn:" + tag, fl_c, _OPS.window_attention_planes, ws[5], ws[3], ws[4], n, half, *gc, None, msg_s)
            else:
                if q_f is None:
                    q_f = f32(c)
                G(blk["tc_q_c"], x1_s, rows=rp, out_f32=q_f)
                msg = self._timed("attn_simt:" + tag, fl_c, _OPS.window_attention, tok(q_f, 0, 128), tok(y, 384, 512), tok(y, 512, 640), half, *gc)
                _OPS.split_planes(msg.view(rows, c), msg_s, 0)
            G(blk["tc_m_c"], msg_s, rows=rp, out_split=m_s)
            # ---- FFN on cat([source, message]) + LayerNorm + residual
            w1, w2 = blk["tc_w1"], blk["tc_w2"]
            if fused_ffn:
                self._timed("conv", 2.0 * rp * hid * (2 * c + c), _OPS.ffn_tc, x1_s, m_s, w1.weights, w2.weights, x1_f,
                            w2.gamma, w2.beta, xo_f, xo_s, rp)
            else:
                G(w1, x1_s, m_s, rows=rp, out_split=hid_s)
                G(w2, hid_s, rows=rp, out_f32=xo_f, out_split=xo_s, aux0=x1_f)
            x_f, xo_f, x_s, xo_s = xo_f, x_f, xo_s, x_s
        return x_f[:rows].view(n, l, c), x_s

    # ------------------------------------------------------------------------------------------ per-scale stages
    def _stage_features(self, f0, f1, flow, h, wd, splits):
        """Warp the second view with the current estimate (unimatch.py:156-168, geometry.py:65-72) and add the per-window
        sine position encoding to both views (utils.py:111-131).  f0, f1: [Bp, h, w, 128]; returns tokens [2Bp, L, 128]."""
        Bp, c = f0.shape[0], f0.shape[-1]
        if flow is not None:
            f1 = _OPS.flow_warp(f1.contiguous(), flow.contiguous(), h, wd)
        table = self._pos_table(h // splits, wd // splits, f0.device)
        tok = torch.cat((f0, f1), dim=0).view(2 * Bp, h, wd, c)
        return _OPS.add_position(tok, table, h, wd).view(2 * Bp, h * wd, c)

    def _stage_correlation(self, tok, Bp, h, wd, task, radius, pred_bidir_flow=False, depth=None):
        """Correlation + softmax (unimatch.py:186-216) on the transformer outputs tok [2Bp, L, 128] -> [ns, h, w, fd]."""
        t0, t1 = tok[:Bp], tok[Bp:]
        if task == "depth":
            cams, from_argmax, bidir = depth                                 # cams: `depth_cameras`
            if bidir:
                q0, q1 = torch.cat((t0, t1), 0).contiguous(), torch.cat((t1, t0), 0).contiguous()
            else:
                q0, q1 = t0.contiguous(), t1.contiguous()
            return _OPS.depth_corr_softmax(q0, q1, cams["K"].contiguous(), cams["K_inv"].contiguous(),
                                           cams["pose"].contiguous(), cams["cand"], h, wd, bool(from_argmax))
        if radius == -1:
            if task == "flow":
                ns = 2 * Bp if pred_bidir_flow else Bp
                return _OPS.softmax_expectation(tok, tok, None, ns, Bp, 2, ops.VALUE_COORDS, ops.POST_MINUS_OWN,
                                                h, wd, 1, 1, ops.MASK_NONE).view(ns, h, wd, 2)
            if task == "stereo":
                return _OPS.softmax_expectation(tok, tok, None, Bp, Bp, 1, ops.VALUE_XCOORD, ops.POST_OWN_MINUS,
                                                h, wd, h, 1, ops.MASK_CAUSAL).view(Bp, h, wd, 1)
            raise NotImplementedError
        if task == "flow":
            return _OPS.local_corr_softmax(t0.contiguous(), t1.contiguous(), h, wd, radius, radius, False)
        if task == "stereo":
            return _OPS.local_corr_softmax(t0.contiguous(), t1.contiguous(), h, wd, 0, radius, True)
        raise NotImplementedError

    def _stage_propagation(self, P, x_s, flow, nb, h, wd, prop_r):
        """SelfAttnPropagation.forward (attention.py:184-253) on the first `nb` streams of the transformer output planes
        x_s [2, rows_padded, 128]: q = Wq x + bq; global: k = Wk q + bk, out = softmax(q k^T / sqrt(C)) flow;
        local (radius r): k = Wk x + bk, 3x3 zero-padded window.  Both projections are wgmma GEMMs."""
        dev = flow.device
        L = h * wd
        rows = nb * L
        rq = rows if rows % 16 == 0 else x_s.shape[1]            # the GEMM runs over a multiple of 16 rows
        G = self._conv
        fd = flow.shape[-1]
        flow = flow.contiguous()
        if prop_r > 0:
            qk = torch.empty((rq, 256), device=dev)
            G(P["prop_qk"], x_s, rows=rq, out_f32=qk)
            qk = qk[:rows].view(nb, L, 256)
            return _OPS.propagate_local(qk[:, :, :128], qk[:, :, 128:], flow, h, wd, prop_r)
        q = torch.empty((rq, 128), device=dev)
        q_s = torch.empty((2, rq, 128), device=dev, dtype=torch.float16)
        k = torch.empty((rq, 128), device=dev)
        G(P["prop_q"], x_s, rows=rq, out_f32=q, out_split=q_s)
        G(P["prop_k"], q_s, rows=rq, out_f32=k)
        return _OPS.softmax_expectation(q[:rows].view(nb, L, 128), k[:rows].view(nb, L, 128), flow.view(nb, L, fd), nb, 0, fd,
                                        ops.VALUE_TENSOR, ops.POST_NONE, h, wd, 1, 1, ops.MASK_NONE).view(nb, h, wd, fd)

    # ------------------------------------------------------------------------------------------ refinement
    class _RefineState:
        pass

    def _stage_refine_setup(self, P, feat0, b, h, w):
        """Loop-invariant part of the refinement (unimatch.py:315-320): net = tanh(.), inp = relu(.) of refine_proj(feature0),
        and the activation planes the update block reuses every iteration.  feat0: [b, h, w, 128] fp32."""
        T = P["tc"]
        dev = feat0.device
        st = self._RefineState()
        z16 = lambda cp: torch.empty((2, b, h, w, cp), device=dev, dtype=torch.float16)
        st.corr_s = self._zero_padded("corr", (2, b, h, w, 128), dev)    # 81 real channels, padding stays zero
        st.cor1_s, st.cf_s, st.flo1_s = z16(256), z16(256), z16(128)
        st.inp_s, st.mfx_s = z16(128), z16(128)                      # inp | (motion features, flow): x of the GRU in two buffers
        st.h0_s, st.h1_s, st.h2_s, st.rh_s, st.fh_s = z16(128), z16(128), z16(128), z16(128), z16(256)
        f0_s = z16(128)
        _OPS.split_planes(feat0, f0_s, 0)
        f32 = lambda cc: torch.empty((b, h, w, cc), device=dev)
        st.net0, st.z, st.h1, st.h2 = f32(128), f32(128), f32(128), f32(128)
        C = self._conv
        C(T["proj_net"], f0_s, out_f32=st.net0, out_split=st.h0_s)
        C(T["proj_inp"], f0_s, out_split=st.inp_s)
        # loop-invariant shares of the four GRU convolutions (bias included), fp32
        st.pre_zr1, st.pre_q1, st.pre_zr2, st.pre_q2 = f32(256), f32(128), f32(256), f32(128)
        C(T["zr1_fix"], st.h0_s, st.inp_s, out_f32=st.pre_zr1)
        C(T["q1_fix"], st.inp_s, out_f32=st.pre_q1)
        C(T["zr2_fix"], st.inp_s, out_f32=st.pre_zr2)
        C(T["q2_fix"], st.inp_s, out_f32=st.pre_q2)
        return st

    def _update_block(self, P, st, corr, flow, want_mask):
        """BasicUpdateBlock.forward (reg_refine.py:106-119) as 11 tensor-core convolutions: activations live as fp16 (hi, lo)
        planes, the concatenations are channel offsets / second sources, the GRU gate math is the conv epilogue."""
        T, w = P["tc"], P["raw"]
        fd = T["fh2"].cout
        C = self._conv
        b, h, wd, _ = corr.shape
        dev = corr.device
        _OPS.split_planes(corr, st.corr_s, 0)
        C(T["convc1"], st.corr_s, out_split=st.cor1_s)
        C(T["convc2"], st.cor1_s, out_split=st.cf_s)
        _OPS.conv7x7_small(flow, None, False, w["refine.encoder.convf1.weight"], w["refine.encoder.convf1.bias"], 1, True,
                           None, None, None, st.flo1_s)        # 7x7 on 1-2 channels: direct fp32 kernel -> fp16 planes
        C(T["convf2"], st.flo1_s, out_split=st.cf_s, off_split=192)
        C(T["conv"], st.cf_s, out_split=st.mfx_s)
        _OPS.split_planes(flow, st.mfx_s, 128 - fd)                              # mfx = [motion features | flow]
        # SepConvGRU (reg_refine.py:37-52): horizontal 1x5 then vertical 5x1; the invariant input channels come in through `pre`
        C(T["zr1_var"], st.mfx_s, out_f32=st.z, out_split=st.rh_s, aux0=st.net0, pre=st.pre_zr1)
        C(T["q1_var"], st.rh_s, st.mfx_s, out_f32=st.h1, out_split=st.h1_s, aux0=st.net0, aux1=st.z, pre=st.pre_q1)
        C(T["zr2_var"], st.h1_s, st.mfx_s, out_f32=st.z, out_split=st.rh_s, aux0=st.h1, pre=st.pre_zr2)
        C(T["q2_var"], st.rh_s, st.mfx_s, out_f32=st.h2, out_split=st.h2_s, aux0=st.h1, aux1=st.z, pre=st.pre_q2)
        C(T["fh1"], st.h2_s, out_split=st.fh_s)
        delta = torch.empty((b, h, wd, fd), device=dev)
        C(T["fh2"], st.fh_s, out_f32=delta)
        mask = None
        if want_mask and "mask0" in T:
            C(T["mask0"], st.h2_s, out_split=st.fh_s)
            mask = torch.empty((b, h, wd, T["mask2"].cout), device=dev)
            C(T["mask2"], st.fh_s, out_f32=mask)
        return st.h2, mask, delta

    def _stage_refine_iter(self, P, rst, g0, g1, flow, task, want_mask, depth=None):
        """One regression-refinement iteration (unimatch.py:272-354): 9x9 correlation volume at the current estimate on the
        pre-transformer features, update block, residual update.  Returns (flow, mask or None)."""
        h, wd = flow.shape[1], flow.shape[2]
        if task == "depth":
            cams, min_depth, max_depth = depth
            cflow = self._rigid_flow(flow, cams["K"].float(), cams["K_inv"].float(), cams["pose"].float(), h, wd)
        else:
            cflow = flow.contiguous()                                       # disparity handled in-kernel
        with self._section("refine_corr_volume"):
            corr = _OPS.local_corr_volume(g0, g1, cflow, h, wd, 4)
        with self._section("refine_update_block"):
            _, mask, delta = self._update_block(P, rst, corr, flow.contiguous(), want_mask)
        if task == "depth":
            flow = (flow - delta).clamp(min=min_depth, max=max_depth)
        else:
            flow = flow + delta
        if task == "stereo":
            flow = flow.clamp(min=0)
        return flow, mask

    def _stage_upsample_learned(self, P, flow2, feat, factor, mult):
        """unimatch.py:81-93 (convex branch): mask = upsampler(cat(flow, feature)) as two tensor-core convolutions
        (3x3 130 -> 256 + ReLU, 1x1 256 -> 9 F^2), then convex upsampling.  flow2: [B,h,w,2]; feat: [B,h,w,128]."""
        U = P["up"]
        b, h, w, _ = feat.shape
        dev = feat.device
        src = self._zero_padded("upsampler", (2, b, h, w, 192), dev)                # [feature 0..127 | flow 128..129 | 0]
        _OPS.split_planes(feat.contiguous(), src, 0)
        _OPS.split_planes(flow2.contiguous(), src, 128)
        mid = torch.empty((2, b, h, w, 256), device=dev, dtype=torch.float16)
        self._conv(U["c0"], src, out_split=mid)
        m = torch.empty((b, h, w, U["c2"].cout), device=dev)
        self._conv(U["c2"], mid, out_f32=m)
        return _OPS.convex_upsample(flow2.contiguous(), m, factor, float(mult))

    @staticmethod
    def _rigid_flow(inv_depth, K, K_inv, pose, h, w):
        """compute_flow_with_depth_pose(1/inv_depth, K, pose) (geometry.py:99-195) on [B,h,w,1] -> [B,h,w,2];
        K_inv = torch.inverse(K), taken once per forward by `depth_cameras`."""
        b = inv_depth.shape[0]
        dev = inv_depth.device
        ys, xs = torch.meshgrid(torch.arange(h, device=dev, dtype=torch.float32),
                                torch.arange(w, device=dev, dtype=torch.float32), indexing="ij")
        grid = torch.stack([xs, ys, torch.ones_like(xs)], dim=0).view(1, 3, -1).expand(b, 3, h * w)
        depth = (1.0 / inv_depth.view(b, 1, h * w))
        pts = K_inv.bmm(grid) * depth
        pts = torch.bmm(pose[:, :3, :3], pts) + pose[:, :3, -1:]
        proj = torch.bmm(K, pts)
        z = proj[:, 2:3].clamp(min=1e-3)
        uv = proj[:, :2] / z - grid[:, :2]
        return uv.view(b, 2, h, w).permute(0, 2, 3, 1).contiguous()

    # ------------------------------------------------------------------------------------------ forward
    def forward(self, img0, img1, attn_type=None, attn_splits_list=None, corr_radius_list=None, prop_radius_list=None,
                num_reg_refine=1, pred_bidir_flow=False, task="flow", intrinsics=None, pose=None,
                min_depth=1. / 0.5, max_depth=1. / 10, num_depth_candidates=64, depth_from_argmax=False,
                pred_bidir_depth=False, **kwargs):
        if self.training:
            raise NotImplementedError("unimatch_b200.UniMatch is inference-only; call .eval()")
        # no device check here: the unimatch_sm100 ops are registered for CUDA only, so CPU tensors fail loudly
        # in the dispatcher (there is no CPU path)
        with torch.no_grad():
            P = self._prepared()
            B = img0.shape[0]
            with self._section("backbone"):                                       # [2B,h,w,128] low -> high res
                feats = self._stage_backbone(P, img0.float().contiguous(), img1.float().contiguous(), task == "flow")
            return self._forward_encoded(P, [f[:B] for f in feats], [f[B:] for f in feats], attn_type, attn_splits_list,
                                         corr_radius_list, prop_radius_list, num_reg_refine, pred_bidir_flow, task, None,
                                         intrinsics, pose, min_depth, max_depth, num_depth_candidates, depth_from_argmax,
                                         pred_bidir_depth)

    # ------------------------------------------------------------------------------------------ depth cameras
    def depth_cameras(self, intrinsics, pose, up, min_depth, max_depth, num_depth_candidates, pred_bidir_depth):
        """The camera operands of the depth task (unimatch.py:176-190, geometry.py:99-195), as a dict of device tensors:
          'Ks'     intrinsics [B,3,3] at the feature resolution (rows 0-1 divided by `up`, the upsample factor);
          'K'      intrinsics of the matched streams: Ks, repeated for the backward streams when `pred_bidir_depth`;
          'K_inv'  torch.inverse(K), read by the depth correlation and by the rigid flow of the refinement;
          'pose'   relative poses of the matched streams: `pose` [B,4,4], with `torch.inverse(pose)` appended when
                   `pred_bidir_depth`; a `pose` of 2B matrices is taken to hold those inverses already (e.g. computed on the
                   host) and is used as it is;
          'cand'   the inverse-depth candidates linspace(min_depth, max_depth, n), built once per (min, max, n, device).
        `forward` builds them after the encoder with the same calls it always made, so its results do not change.  The
        stages only read them: given `cameras`, `forward_encoded` issues no host synchronisation and no pageable copy and can
        be captured in a CUDA graph.  `torch.inverse` checks its result on the host, so build the cameras outside a capture."""
        dev = intrinsics.device
        Ks = intrinsics.clone().float()
        Ks[:, :2] = Ks[:, :2] / up
        B = Ks.shape[0]
        if pred_bidir_depth:
            K = Ks.repeat(2, 1, 1)
            pc = pose.float() if pose.shape[0] == 2 * B else torch.cat((pose, torch.inverse(pose)), dim=0).float()
        else:
            K, pc = Ks, pose.float()
        key = (float(min_depth), float(max_depth), int(num_depth_candidates), str(dev))
        cand = self._cands.get(key)
        if cand is None:
            cand = self._cands[key] = torch.linspace(min_depth, max_depth, num_depth_candidates).float().to(dev)   # :190
        return {"Ks": Ks, "K": K, "K_inv": torch.inverse(K), "pose": pc, "cand": cand}

    # ------------------------------------------------------------------------------------------ video: encode frames once
    def encode_frames(self, frames, task="flow"):
        """CNN encoder on a set of frames [T,3,H,W]: in [0,255] for the flow task (normalize_img folded into the stem), already
        ImageNet-normalised for stereo and depth, as `forward` takes them for each task.  Returns the feature
        pyramid low -> high resolution, each [T,h,w,128].  Every encoder kernel works per image (convolutions per pixel,
        InstanceNorm per image over a fixed chunking), so a frame's features do not depend on its partner or on the batch and
        consecutive pairs of a video can share one encoding per frame.  They are equal up to fp32 summation order, not bit
        for bit: um_conv2d_tc walks the K chunks of an output tile in an order rotated by the index of the CTA that owns the
        tile (to spread the weight reads over L2), and the tile-to-CTA assignment follows the launch's tile count, so the
        same frame in a batch of a different size can round differently in the last bits."""
        if self.training:
            raise NotImplementedError("unimatch_b200.UniMatch is inference-only; call .eval()")
        if task not in ("flow", "stereo", "depth"):
            raise ValueError("encode_frames: unknown task %r" % (task,))
        with torch.no_grad():
            P = self._prepared()
            with self._section("backbone"):
                return self._stage_backbone(P, frames.float().contiguous(), None, task == "flow")

    def forward_encoded(self, feats0, feats1, attn_type=None, attn_splits_list=None, corr_radius_list=None,
                        prop_radius_list=None, num_reg_refine=1, pred_bidir_flow=False, task="flow", cameras=None,
                        intrinsics=None, pose=None, min_depth=1. / 0.5, max_depth=1. / 10, num_depth_candidates=64,
                        depth_from_argmax=False, pred_bidir_depth=False, **kwargs):
        """Everything of `forward` after the encoder, on per-scale features of the first and second views ([B,h,w,128] each,
        low -> high resolution, e.g. slices `f[:-1]`, `f[1:]` of `encode_frames`).  Returns {'flow_preds': [...]} exactly as
        `forward` does for the images those features were encoded from (encoded with `encode_frames(..., task)`).
        Flow and depth.  Depth: `cameras` = `depth_cameras(...)` for these B pairs (then `intrinsics`, `pose` and
        `num_depth_candidates` are not read, and nothing here synchronises with the host), or `intrinsics` and `pose` as
        `forward` takes them.  Stereo is not offered: its pairs share no view, so there is no encoding to reuse.
        A caller who captures this call (or `forward`) in a CUDA graph of their own must keep the tensors of
        `cached_buffers()`, taken just after the capture, for as long as they replay the graph: calls at other batch sizes or
        shapes can evict them from the module's caches, and a replay would then write into memory another tensor owns."""
        if self.training:
            raise NotImplementedError("unimatch_b200.UniMatch is inference-only; call .eval()")
        if task not in ("flow", "depth"):
            raise ValueError("forward_encoded drives the flow and depth tasks only (each stereo pair encodes two distinct views)")
        if len(feats0) != self.num_scales or len(feats1) != self.num_scales:
            raise ValueError("forward_encoded needs one feature map per scale (%d)" % self.num_scales)
        with torch.no_grad():
            return self._forward_encoded(self._prepared(), list(feats0), list(feats1), attn_type, attn_splits_list,
                                         corr_radius_list, prop_radius_list, num_reg_refine, pred_bidir_flow, task, cameras,
                                         intrinsics, pose, min_depth, max_depth, num_depth_candidates, depth_from_argmax,
                                         pred_bidir_depth)

    def _forward_encoded(self, P, feats0, feats1, attn_type, attn_splits_list, corr_radius_list, prop_radius_list,
                         num_reg_refine, pred_bidir_flow, task, cams, intrinsics, pose, min_depth, max_depth,
                         num_depth_candidates, depth_from_argmax, pred_bidir_depth):
        """The per-task argument checks of `forward` and `forward_encoded`, then the matching path after the encoder
        (unimatch.py:127-367).  feats0 / feats1: per-scale [B,h,w,128] views; cams: `depth_cameras` for the depth task, or
        None to build them here from `intrinsics` and `pose`."""
        assert task == "flow" or not pred_bidir_flow
        if task == "depth":
            assert self.num_scales == 1 and len(attn_splits_list) == len(prop_radius_list) == 1
            if cams is None:
                if intrinsics is None or pose is None:
                    raise ValueError("the depth task needs intrinsics= and pose= (or, in forward_encoded, cameras=)")
                cams = self.depth_cameras(intrinsics, pose, self.upsample_factor, min_depth, max_depth, num_depth_candidates,
                                          pred_bidir_depth)
            streams = (2 if pred_bidir_depth else 1) * feats0[0].shape[0]
            if cams["K"].shape[0] != streams or cams["pose"].shape[0] != streams:
                raise ValueError("the depth cameras were built for another batch or pred_bidir_depth setting")
        else:
            assert len(attn_splits_list) == len(corr_radius_list) == len(prop_radius_list) == self.num_scales
            cams, pred_bidir_depth, depth_from_argmax = None, False, False
        flow = None            # [Bp, h, w, fd] channel-last
        preds = []
        for s in range(self.num_scales):
            f0, f1 = feats0[s], feats1[s]
            _, h, wd, c = f0.shape
            if pred_bidir_flow and s > 0:                                         # unimatch.py:139-141
                f0, f1 = torch.cat((f0, f1), dim=0), torch.cat((f1, f0), dim=0)
            f0_ori, f1_ori = f0, f1
            Bp = f0.shape[0]
            if s > 0:
                flow = _OPS.upsample2x(flow.contiguous(), 2.0)                    # unimatch.py:154
            splits = attn_splits_list[s]
            prop_r = prop_radius_list[s]
            tok = self._stage_features(f0, f1, flow, h, wd, splits)
            with self._section("transformer_s%d" % s):
                tok, tok_s = self._stage_transformer(P, tok, h, wd, attn_type, splits, "s%d" % s)   # [2Bp, L, 128]

            # ---- correlation + softmax (unimatch.py:186-216) ----
            with self._section("correlation_s%d" % s):
                dargs = (cams, depth_from_argmax, pred_bidir_depth) if task == "depth" else None
                pred = self._stage_correlation(tok, Bp, h, wd, task, None if task == "depth" else corr_radius_list[s],
                                               pred_bidir_flow, dargs)
            flow = flow + pred if flow is not None else pred
            if task == "stereo":
                flow = flow.clamp(min=0)

            # ---- self-attention propagation (unimatch.py:230-237, attention.py:184-253) ----
            bidir0 = (pred_bidir_flow or pred_bidir_depth) and s == 0
            nb = 2 * Bp if bidir0 else Bp                                         # bidirectional: cat(feature0, feature1)
            with self._section("propagation_s%d" % s):
                flow = self._stage_propagation(P, tok_s, flow, nb, h, wd, prop_r)
            if s != self.num_scales - 1:
                continue

            feat0 = tok[:nb].reshape(nb, h, wd, c)                                # post-transformer feature0
            # ---- regression refinement (unimatch.py:272-354) ----
            if self.reg_refine:
                assert num_reg_refine > 0
                g0, g1 = f0_ori.contiguous(), f1_ori.contiguous()
                drefine = None
                if task == "depth":
                    if pred_bidir_depth:
                        g0, g1 = torch.cat((g0, g1), dim=0), torch.cat((g1, g0), dim=0)
                    drefine = (cams, min_depth, max_depth)
                rst = self._stage_refine_setup(P, feat0.contiguous(), nb, h, wd)
                for it in range(num_reg_refine):
                    flow, mask = self._stage_refine_iter(P, rst, g0, g1, flow, task, it == num_reg_refine - 1, drefine)

            # ---- upsampling to the input resolution (unimatch.py:246-264; after the refinement :335-354) ----
            up = self.upsample_factor
            if task == "depth":
                out = self._stage_upsample_learned(P, torch.cat((flow, torch.zeros_like(flow)), -1), feat0, up,
                                                   1).clamp(min=min_depth, max=max_depth)[:, :1]
            elif self.reg_refine:
                out = _OPS.convex_upsample(flow.contiguous(), mask, up, float(up))
            elif task == "stereo":
                out = -self._stage_upsample_learned(P, torch.cat((-flow, torch.zeros_like(flow)), -1), feat0, up, up)[:, :1]
            else:
                out = self._stage_upsample_learned(P, flow, feat0, up, up)
            preds.append(out)

        if task == "stereo":
            preds = [p.squeeze(1) for p in preds]
        if task == "depth":
            preds = [1.0 / p.squeeze(1) for p in preds]
        return {"flow_preds": preds}
