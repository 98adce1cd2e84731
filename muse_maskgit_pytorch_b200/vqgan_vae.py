"""VQGanVAE — host-side mirror of the reference class (ref: vqgan_vae.py:285-463) over libmmg.so.

Same constructor keywords, attribute names, state_dict keys and method signatures as the reference for the inference
surface (encode / decode / decode_from_ids / forward without losses / get_encoded_fmap_size / copy_for_eval / save / load).
The modules below only HOLD parameters under the reference's key names; all arithmetic happens in the sm_90a kernels:
convolutions are implicit GEMMs over NHWC activations (wgmma + TMA in bf16 precision, or e4m3 operands with per-image and per-row
scales under precision="fp8"), the quantizer is the LFQ sign
scan / explicit L2 argmin scan.  Training losses (GAN, VGG; vqgan_vae.py:350-385, 465-534) are out of scope.
"""
import copy
import math
from pathlib import Path

import torch
from torch import nn

from . import ops, pack_cache

# conv-transpose (k4, s2, p1) parity classes: output row 2y+py reads kernel rows CT_R[py][a] at input offsets CT_D[py][a]
CT_R = ((1, 3), (0, 2))
CT_D = ((0, -1), (1, 0))


def _prefixed(prefix, d):
    hit = {k[len(prefix):]: v for k, v in d.items() if k.startswith(prefix)}
    rest = {k: v for k, v in d.items() if not k.startswith(prefix)}
    return hit, rest


class _Net(nn.Module):
    """Parameter holder exposing children under `.net.<i>` like the reference's res-blocks."""
    def __init__(self, layers):
        super().__init__()
        self.net = nn.Sequential(*layers)


class _EncDec(nn.Module):
    """Parameter layout of the reference ResnetEncDec (vqgan_vae.py:185-232): same module order, hence the same state_dict keys, for any
    `layers`, `layer_mults`, `num_resnet_blocks` (int or per-stage tuple) and odd `first_conv_kernel_size`.  `enc_plan` / `dec_plan` list
    what each entry of `encoders` / `decoders` is, in execution order."""
    def __init__(self, dim, channels=3, layers=4, layer_mults=None, num_resnet_blocks=1, resnet_groups=16,
                 first_conv_kernel_size=5):
        super().__init__()
        assert dim % resnet_groups == 0, f"dimension {dim} must be divisible by {resnet_groups} (groups for the groupnorm)"
        assert first_conv_kernel_size % 2 == 1 and 1 <= first_conv_kernel_size <= 9, \
            "first_conv_kernel_size must be odd (the reference pads by kernel_size // 2, vqgan_vae.py:231) and at most 9 here"
        self.layers, self.groups, self.first_k = layers, resnet_groups, first_conv_kernel_size
        mults = layer_mults if layer_mults is not None else [2 ** i for i in range(layers)]
        assert len(mults) == layers, "layer multipliers must be equal to designated number of layers"
        dims = [dim] + [dim * m for m in mults]
        self.dims = dims
        self.encoded_dim = dims[-1]
        if not isinstance(num_resnet_blocks, tuple):
            num_resnet_blocks = (0,) * (layers - 1) + (num_resnet_blocks,)
        assert len(num_resnet_blocks) == layers, "number of resnet blocks config must be equal to number of layers"
        act = lambda: nn.LeakyReLU(0.1)
        enc, dec = [], []
        for cin, cout, nres in zip(dims[:-1], dims[1:], num_resnet_blocks):
            enc.append(nn.Sequential(nn.Conv2d(cin, cout, 4, stride=2, padding=1), act()))
            dec.insert(0, nn.Sequential(nn.ConvTranspose2d(cout, cin, 4, 2, 1), act()))
            for _ in range(nres):
                enc.append(_Net([nn.Conv2d(cout, cout, 3, padding=1), nn.GroupNorm(resnet_groups, cout), act(),
                                 nn.Conv2d(cout, cout, 3, padding=1), nn.GroupNorm(resnet_groups, cout), act(), nn.Conv2d(cout, cout, 1)]))
                dec.insert(0, _Net([nn.Conv2d(cout, 2 * cout, 3, padding=1), nn.GLU(dim=1), nn.GroupNorm(resnet_groups, cout),
                                    nn.Conv2d(cout, 2 * cout, 3, padding=1), nn.GLU(dim=1), nn.GroupNorm(resnet_groups, cout),
                                    nn.Conv2d(cout, cout, 1)]))
        enc.insert(0, nn.Conv2d(channels, dim, first_conv_kernel_size, padding=first_conv_kernel_size // 2))
        dec.append(nn.Conv2d(dim, channels, 1))
        self.encoders, self.decoders = nn.ModuleList(enc), nn.ModuleList(dec)

        def plan(mods, plain):
            out = []
            for i, mod in enumerate(mods):
                if isinstance(mod, _Net):
                    out.append(("glu" if isinstance(mod.net[1], nn.GLU) else "res", i, mod.net[0].in_channels))
                elif isinstance(mod, nn.Sequential):
                    conv = mod[0]
                    out.append(("up" if isinstance(conv, nn.ConvTranspose2d) else "down", i, conv.in_channels, conv.out_channels))
                else:
                    out.append((plain, i))          # the k x k stem of the encoder / the final 1x1 conv of the decoder
            return out
        self.enc_plan, self.dec_plan = plan(self.encoders, "in"), plan(self.decoders, "rgb")
        assert self.enc_plan[0][0] == "in" and self.dec_plan[-1][0] == "rgb"
        self.has_res = any(e[0] == "res" for e in self.enc_plan)

    def get_encoded_fmap_size(self, image_size):
        return image_size // (2 ** self.layers)


class _LFQ(nn.Module):
    """Parameter layout of vector_quantize_pytorch.LFQ (inference): project_in / project_out / mask buffer."""
    def __init__(self, dim, codebook_size):
        super().__init__()
        bits = int(math.log2(codebook_size))
        assert 2 ** bits == codebook_size, "LFQ needs a power-of-two codebook"
        self.bits = bits
        self.project_in = nn.Linear(dim, bits) if dim != bits else nn.Identity()
        self.project_out = nn.Linear(bits, dim) if dim != bits else nn.Identity()
        self.register_buffer("mask", 2 ** torch.arange(bits - 1, -1, -1))


class _EuclideanVQ(nn.Module):
    """Explicit codebook (the path the reference intends at vqgan_vae.py:337-342, defect B1 fixed): codebook_dim == dim."""
    def __init__(self, dim, codebook_size):
        super().__init__()
        self.embed = nn.Parameter(torch.randn(codebook_size, dim))

    @property
    def codebook(self):
        return self.embed


class VQGanVAE(nn.Module):
    def __init__(self, *, dim, channels=3, layers=4, l2_recon_loss=False, use_hinge_loss=True, vgg=None,
                 lookup_free_quantization=True, codebook_size=65536, vq_kwargs: dict = None, lfq_kwargs: dict = None,
                 use_vgg_and_gan=True, discr_layers=4, precision=None, **kwargs):
        super().__init__()
        vq_kw, kwargs = _prefixed("vq_", kwargs)
        encdec_kw, kwargs = _prefixed("encdec_", kwargs)
        self.channels, self.codebook_size, self.dim_divisor = channels, codebook_size, 2 ** layers
        self.enc_dec = _EncDec(dim=dim, channels=channels, layers=layers, **encdec_kw)
        self.lookup_free_quantization = lookup_free_quantization
        D = self.enc_dec.encoded_dim
        self.quantizer = _LFQ(D, codebook_size) if lookup_free_quantization else _EuclideanVQ(D, codebook_size)
        self.use_vgg_and_gan = False          # no discriminator / VGG in this inference build (dropped by copy_for_eval in the reference)
        self.discr, self._vgg = None, None
        self.precision = precision or "bf16"
        if self.precision == "fp8":
            # e4m3 convolutions take one k-block per tap and 128 input channels: every conv / conv-transpose input width must be a multiple
            # of 128 (the stem conv_in and the final 1x1 RGB conv stay as they are)
            for w in self._conv_input_widths():
                if w % 128:
                    raise ValueError(f'VQGanVAE precision="fp8" needs every conv input width to be a multiple of 128; this model has a conv '
                                     f'with {w} input channels (use precision="bf16")')
        self._pack = None
        # both hooks also fire when a PARENT module (MaskGit, Muse) loads a checkpoint: checkpoints written by the reference carry
        # discriminator / VGG tensors (vqgan_vae.py:344-348, dropped by copy_for_eval :394-403) that are not part of inference
        self._register_load_state_dict_pre_hook(self._drop_training_only_keys)
        self.register_load_state_dict_post_hook(lambda m, _inc: setattr(m, "_pack", None))

    @staticmethod
    def _drop_training_only_keys(state_dict, prefix, *_):
        for k in [k for k in state_dict if k.startswith((prefix + "discr.", prefix + "_vgg."))]:
            del state_dict[k]

    def _conv_input_widths(self):
        """input channels of every conv and conv-transpose the implicit-GEMM kernels run (not the stem conv_in nor the final 1x1)"""
        ed = self.enc_dec
        return [e[2] for e in ed.enc_plan + ed.dec_plan if e[0] in ("down", "res", "glu", "up")]

    def _weights_sig(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _check_weights(self):
        if self._pack is not None and self._pack.get("sig") != self._weights_sig():
            self._pack = None

    # ----- reference surface ------------------------------------------------------------------------------------
    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def encoded_dim(self):
        return self.enc_dec.encoded_dim

    @property
    def codebook(self):
        return self.quantizer.codebook

    def get_encoded_fmap_size(self, image_size):
        return self.enc_dec.get_encoded_fmap_size(image_size)

    def copy_for_eval(self):
        """ref: vqgan_vae.py:394-403 — an eval copy without training-only parts (the caller's module is left in place)."""
        c = copy.deepcopy(self)
        c._pack = None
        return c.eval()

    def save(self, path):
        torch.save(self.state_dict(), path)

    def load(self, path):
        path = Path(path)
        assert path.exists()
        self.load_state_dict(torch.load(str(path)))

    def _apply(self, fn, *a, **k):
        self._pack = None
        return super()._apply(fn, *a, **k)

    # ----- weight packing ---------------------------------------------------------------------------------------
    def _adt(self):
        """activation dtype: bf16 for "bf16" and "fp8" (e4m3 is only the operand type of the convolutions), fp32 for "fp32\""""
        return torch.bfloat16 if self.precision in ("bf16", "fp8") else torch.float32

    def _packed(self):
        if self._pack is not None and self._pack["adt"] == self._adt() and self._pack.get("fp8", False) == (self.precision == "fp8"):
            return self._pack
        dev = self.device
        assert dev.type == "cuda", "VQGanVAE runs on CUDA only (libmmg.so); there is no CPU path"
        P = pack_cache.load_or_build("vqgan_vae", self, (self.precision, self.lookup_free_quantization), self._build_pack, dev)
        P["sig"] = self._weights_sig()
        self._pack = P
        return P

    def _build_pack(self):
        adt, dev = self._adt(), self.device
        fp8 = self.precision == "fp8"
        P = {"adt": adt, "fp8": fp8}
        ed, L = self.enc_dec, self.enc_dec.layers
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()
        # (Cout,kh,kw,Cin); fp8 keeps fp32 here and quantises the finished row layout in `wq`
        conv_w = lambda w: w.detach().permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(dev, torch.float32 if fp8 else adt).contiguous()

        def wq(w2d):
            """the operand the conv kernels take: the packed weight itself, or (fp8) its e4m3 rows and one fp32 scale per output row"""
            if not fp8:
                return w2d
            from .muse_maskgit import quantize_rows_e4m3
            return quantize_rows_e4m3(w2d)

        def glu_interleave(w2d, bias):         # rows [a(32) | gate(32)] per block so the epilogue sees both halves of a unit
            C2 = w2d.shape[0]; Cc = C2 // 2
            assert Cc % 32 == 0, ("GLUResBlock channels must be a multiple of 32 here (the gate and value halves are interleaved in blocks of 32 output "
                                  "channels for the fused conv + GLU epilogue); the reference takes any width divisible by resnet_groups (vqgan_vae.py:251-265)")
            idx = torch.arange(Cc, device=w2d.device).view(-1, 32)
            order = torch.cat((idx, idx + Cc), dim=1).reshape(-1)
            return w2d[order].contiguous(), bias[order].contiguous()

        P["e0_w"], P["e0_b"] = f32(ed.encoders[0].weight), f32(ed.encoders[0].bias)
        P["enc"], P["dec"] = {}, {}                                     # module index -> packed tensors, following enc_plan / dec_plan
        for kind, i, *_ in ed.enc_plan:
            if kind == "down":
                P["enc"][i] = (wq(conv_w(ed.encoders[i][0].weight)), f32(ed.encoders[i][0].bias))
            elif kind == "res":
                n = ed.encoders[i].net
                P["enc"][i] = dict(w1=wq(conv_w(n[0].weight)), b1=f32(n[0].bias), g1=f32(n[1].weight), be1=f32(n[1].bias),
                                   w2=wq(conv_w(n[3].weight)), b2=f32(n[3].bias), g2=f32(n[4].weight), be2=f32(n[4].bias),
                                   w3=wq(conv_w(n[6].weight)), b3=f32(n[6].bias))
        for kind, i, *_ in ed.dec_plan:
            if kind == "glu":
                n = ed.decoders[i].net
                w1, b1 = glu_interleave(conv_w(n[0].weight), f32(n[0].bias))
                w2, b2 = glu_interleave(conv_w(n[3].weight), f32(n[3].bias))
                P["dec"][i] = dict(w1=wq(w1), b1=b1, g1=f32(n[2].weight), be1=f32(n[2].bias), w2=wq(w2), b2=b2, g2=f32(n[5].weight),
                                   be2=f32(n[5].bias), w3=wq(conv_w(n[6].weight)), b3=f32(n[6].bias))
            elif kind == "up":
                ct = ed.decoders[i][0]
                w = ct.weight.detach().to(dev, torch.float32)                 # (Cin, Cout, 4, 4)
                packs = []
                for py in range(2):
                    for px in range(2):
                        taps = [w[:, :, CT_R[py][a], CT_R[px][b]].t() for a in range(2) for b in range(2)]   # each (Cout, Cin)
                        packs.append(torch.cat(taps, dim=1))
                st = torch.stack(packs)                                        # [4 parities, Cout, 4 Cin]
                if fp8:                                                        # one scale per row of each parity stack: [4, Cout]
                    q, s = wq(st.reshape(-1, st.shape[2]))
                    P["dec"][i] = ((q.view(st.shape).contiguous(), s.view(4, -1).contiguous()), f32(ct.bias))
                else:
                    P["dec"][i] = (st.to(adt).contiguous(), f32(ct.bias))
        last = ed.decoders[-1]
        P["rgb_w"], P["rgb_b"] = f32(last.weight.reshape(last.weight.shape[0], -1)), f32(last.bias)
        P["rgb_w_adt"] = P["rgb_w"].to(adt).contiguous()
        q = self.quantizer
        if self.lookup_free_quantization:
            lin = isinstance(q.project_in, nn.Linear)
            P["pin_w"], P["pin_b"] = (f32(q.project_in.weight), f32(q.project_in.bias)) if lin else (None, None)
            P["pout_w"], P["pout_b"] = (f32(q.project_out.weight), f32(q.project_out.bias)) if lin else (None, None)
            P["pin_w3"] = None
            if lin and adt == torch.bfloat16 and 3 * q.bits <= 64 and self.enc_dec.encoded_dim % 64 == 0:
                # project_in split into three bf16 terms (hi + mid + lo reproduces the fp32 weight to 24 bits) stacked as the 64 rows of
                # one wgmma GEMM; the LFQ_IDS epilogue recombines them, adds the bias, takes signs and packs the id
                w = P["pin_w"]
                hi = w.to(adt); r1 = w - hi.float(); mid = r1.to(adt); lo = (r1 - mid.float()).to(adt)
                w3 = torch.zeros((64, w.shape[1]), device=dev, dtype=adt)
                w3[:q.bits], w3[q.bits:2 * q.bits], w3[2 * q.bits:3 * q.bits] = hi, mid, lo
                P["pin_w3"] = w3.contiguous()
        else:
            P["codebook"] = f32(q.embed)
            cb = P["codebook"]
            if adt == torch.bfloat16:
                # the fp32 codebook as three bf16 terms along K, smallest first ([lo | mid | hi], each [codes, D]): against the token repeated
                # three times one bf16 product accumulates x . (lo + mid + hi) = x . e in fp32 — the nearest-code argmin then sees the fp32
                # codebook (the bf16-rounded one misplaced near-ties), at 3x the FLOPs of a lookup that is HBM-bound anyway
                hi = cb.to(adt); r1 = cb - hi.float(); mid = r1.to(adt); lo = (r1 - mid.float()).to(adt)
                P["codebook_a"] = torch.cat((lo, mid, hi), dim=1).contiguous()
            else:
                P["codebook_a"] = cb                                   # fp32: ops.linear splits both operands (mmg_split3)
            P["code_norms"] = (cb * cb).sum(-1).contiguous()
        return P

    # ----- NHWC pipelines (all arithmetic in libmmg) ---------------------------------------------------------------
    @staticmethod
    def _conv(x, w, out, B, H, W, Cin, Cout, kind, **epi):
        """one convolution of the pipelines; w is a packed bf16 / fp32 weight, or (fp8) the pair (e4m3 rows, row scales): the input map is
        then quantised per image for this conv alone"""
        if isinstance(w, tuple):
            VQGanVAE._check_fp8_grid(*((H // 2, W // 2) if kind == 2 else (H, W)))
            q, s = ops.quantize_e4m3_images(x, B)
            return ops.conv2d_fp8(q, s, w[0], w[1], out, B, H, W, Cin, Cout, kind, **epi)
        return ops.conv2d(x, w, out, B, H, W, Cin, Cout, kind, **epi)

    @staticmethod
    def _conv_t(x, w, out, B, H, W, Cin, Cout, **epi):
        if isinstance(w, tuple):
            VQGanVAE._check_fp8_grid(H, W)
            q, s = ops.quantize_e4m3_images(x, B)
            return ops.conv_transpose2d_fp8(q, s, w[0], w[1], out, B, H, W, Cin, Cout, **epi)
        return ops.conv_transpose2d(x, w, out, B, H, W, Cin, Cout, **epi)

    def _encode_nhwc(self, img):
        """img (B,C,H,W) fp32 -> fmap NHWC [B*f*f, D] in activation dtype.  ref: vqgan_vae.py:241-244"""
        P, ed = self._packed(), self.enc_dec
        adt, dev = P["adt"], img.device
        B, C, H, W = img.shape
        img = img.to(torch.float32).contiguous()
        x = torch.empty((B * H * W, ed.dims[0]), device=dev, dtype=adt)
        ops.conv_in(img, P["e0_w"], P["e0_b"], x, ksize=ed.first_k)
        h, w = H, W
        for kind, i, *cc in ed.enc_plan[1:]:
            if kind == "down":
                cin, cout = cc
                cw, cb = P["enc"][i]
                y = torch.empty((B * (h // 2) * (w // 2), cout), device=dev, dtype=adt)
                self._conv(x, cw, y, B, h, w, cin, cout, kind=2, bias=cb, act=1)
                x, h, w = y, h // 2, w // 2
            else:                                   # ResBlock (vqgan_vae.py:267-281)
                R, D = P["enc"][i], cc[0]
                t1 = torch.empty_like(x); t2 = torch.empty_like(x); out = torch.empty_like(x)
                self._conv(x, R["w1"], t1, B, h, w, D, D, kind=1, bias=R["b1"])
                ops.groupnorm_(t1, R["g1"], R["be1"], B, h * w, D, ed.groups, act=1)
                self._conv(t1, R["w2"], t2, B, h, w, D, D, kind=1, bias=R["b2"])
                ops.groupnorm_(t2, R["g2"], R["be2"], B, h * w, D, ed.groups, act=1)
                self._conv(t2, R["w3"], out, B, h, w, D, D, kind=0, epilogue=ops.EPI_RESIDUAL, bias=R["b3"], resid=x)
                x = out
        return x, h, w

    def _decode_nhwc(self, x, B, h, w):
        """fmap NHWC [B*h*w, D] -> images (B, C, H, W) fp32.  ref: vqgan_vae.py:246-249"""
        P, ed = self._packed(), self.enc_dec
        adt, dev = P["adt"], x.device
        plan = ed.dec_plan
        for pi, (kind, i, *cc) in enumerate(plan[:-1]):
            if kind == "glu":                       # GLUResBlock (vqgan_vae.py:251-265)
                R, D = P["dec"][i], cc[0]
                t1 = torch.empty_like(x); t2 = torch.empty_like(x); out = torch.empty_like(x)
                self._conv(x, R["w1"], t1, B, h, w, D, 2 * D, kind=1, epilogue=ops.EPI_GLU, bias=R["b1"])
                ops.groupnorm_(t1, R["g1"], R["be1"], B, h * w, D, ed.groups)
                self._conv(t1, R["w2"], t2, B, h, w, D, 2 * D, kind=1, epilogue=ops.EPI_GLU, bias=R["b2"])
                ops.groupnorm_(t2, R["g2"], R["be2"], B, h * w, D, ed.groups)
                self._conv(t2, R["w3"], out, B, h, w, D, D, kind=0, epilogue=ops.EPI_RESIDUAL, bias=R["b3"], resid=x)
                x = out
                continue
            cin, cout = cc                          # ConvTranspose2d(4, 2, 1) + LeakyReLU
            cw, cb = P["dec"][i]
            last = pi == len(plan) - 2              # directly followed by the final 1x1 conv: fuse both (the full-resolution map stays on chip)
            fuse_rgb = last and adt == torch.bfloat16 and cout in (64, 128, 256) and cin % 64 == 0 and self._tc_tile_ok(h, w)
            if fuse_rgb:
                img = torch.empty((B, self.channels, 2 * h, 2 * w), device=dev, dtype=torch.float32)
                self._conv_t(x, cw, img, B, h, w, cin, cout, bias=cb, rgb_w=P["rgb_w"], rgb_b=P["rgb_b"])
                return img
            y = torch.empty((B * 4 * h * w, cout), device=dev, dtype=adt)
            self._conv_t(x, cw, y, B, h, w, cin, cout, bias=cb)
            x, h, w = y, 2 * h, 2 * w
        rgb = torch.empty((B * h * w, self.channels), device=dev, dtype=torch.float32)
        ops.linear(x, P["rgb_w_adt"], rgb, bias=P["rgb_b"])
        return rgb.view(B, h, w, self.channels).permute(0, 3, 1, 2).contiguous()

    @staticmethod
    def _check_fp8_grid(h, w):
        """the e4m3 convolutions have no CUDA-core kernel behind them: each conv's output grid (conv-transpose: input grid) must have a
        conv tile geometry, which holds for square power-of-two image sizes and for most multiples of 128 pixels"""
        if not VQGanVAE._tc_tile_ok(h, w):
            raise ValueError(f'VQGanVAE precision="fp8": a {h} x {w} feature map has no tile geometry for the e4m3 convolutions (the tile '
                             f'width min(W, 128) must divide 128 and W, and min(128 / width, H) must divide H); use precision="bf16" for '
                             f'this image size')

    @staticmethod
    def _tc_tile_ok(h, w):
        tw = min(w, 128)
        if 128 % tw or w % tw:
            return False
        th = min(128 // tw, h)
        return h % th == 0 and 128 % (tw * th) == 0

    def _quantize_nhwc(self, x):
        P = self._packed()
        ids = torch.empty((x.shape[0],), device=x.device, dtype=torch.int64)
        if self.lookup_free_quantization:
            # bf16 fmap + split projection: wgmma route inside mmg_vq_lfq_encode (HBM-bound TMA stream of the fmap); else CUDA cores
            ops.vq_lfq_encode(x, P["pin_w"], P["pin_b"], ids, self.quantizer.bits, w_split=P["pin_w3"] if x.dtype == torch.bfloat16 else None)
        else:
            ids.fill_(-1)                                   # all-ones keys for the packed (distance, code) atomicMin
            if x.dtype == torch.bfloat16:
                x = torch.cat((x, x, x), dim=1)             # against [lo | mid | hi] of the fp32 codebook
            ops.linear(x, P["codebook_a"], ids, epilogue=ops.EPI_ARGMIN, bias=P["code_norms"])
            ids &= 0xFFFFFFFF
        return ids

    def _codes_nhwc(self, ids_flat):
        P = self._packed()
        D = self.enc_dec.encoded_dim
        if self.lookup_free_quantization:
            out = torch.empty((ids_flat.numel(), D), device=ids_flat.device, dtype=P["adt"])
            ops.vq_decode_codes(ids_flat, P["pout_w"], P["pout_b"], out, self.quantizer.bits)
            return out
        return P["codebook"][ids_flat].to(P["adt"]).contiguous()     # project_out is Identity (codebook_dim == dim)

    # ----- public API ---------------------------------------------------------------------------------------------
    @torch.no_grad()
    def encode(self, fmap):
        """ref: vqgan_vae.py:422-425 — returns (quantized fmap (B,D,f,f) fp32, ids (B,f,f) int64, aux loss 0)."""
        B = fmap.shape[0]
        x, h, w = self._encode_nhwc(fmap)
        ids = self._quantize_nhwc(x)
        q = self._codes_nhwc(ids)
        fq = q.view(B, h, w, -1).permute(0, 3, 1, 2).to(torch.float32).contiguous()
        return fq, ids.view(B, h, w), torch.zeros((), device=fmap.device)

    @torch.no_grad()
    def encode_ids(self, img):
        """ids only (what MaskGit needs for conditioning images); skips the quantized-fmap materialisation."""
        x, h, w = self._encode_nhwc(img)
        return self._quantize_nhwc(x).view(img.shape[0], h, w)

    @torch.no_grad()
    def decode_from_ids(self, ids):
        """ref: vqgan_vae.py:427-438."""
        B, h, w = ids.shape
        x = self._codes_nhwc(ids.reshape(-1).contiguous())
        return self._decode_nhwc(x, B, h, w)

    @torch.no_grad()
    def decode(self, fmap):
        """ref: vqgan_vae.py:440-441 — fmap (B,D,h,w) -> images."""
        B, D, h, w = fmap.shape
        x = fmap.permute(0, 2, 3, 1).reshape(B * h * w, D).to(self._adt()).contiguous()
        return self._decode_nhwc(x, B, h, w)

    @torch.no_grad()
    def forward(self, img, return_loss=False, return_discr_loss=False, return_recons=False, add_gradient_penalty=True):
        """ref: vqgan_vae.py:443-463 (no-loss branch)."""
        B, C, H, W = img.shape
        for name, size in (("height", H), ("width", W)):
            assert size % self.dim_divisor == 0, f"{name} must be divisible by {self.dim_divisor}"
        assert C == self.channels, "number of channels on image or sketch is not equal to the channels set on this VQGanVAE"
        if return_loss or return_discr_loss:
            raise NotImplementedError("VQGanVAE training losses are outside the scope of this inference path")
        x, h, w = self._encode_nhwc(img)
        ids = self._quantize_nhwc(x)
        return self._decode_nhwc(self._codes_nhwc(ids), B, h, w)
