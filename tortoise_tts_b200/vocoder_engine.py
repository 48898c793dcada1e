"""UnivNet vocoder on the sm_90a kernels (hot loop 3, SURVEY §8 row a13).

Mirrors `UnivNetGenerator.inference(c, z)` (tortoise/models/vocoder.py:300-312). Weight-norm is folded at load
time (`remove_weight_norm`, vocoder.py:290-298). The kernel-predictor's kernel_conv + bias_conv become ONE wgmma
GEMM whose rows are permuted so that its output is directly the per-frame kernel block the fused LVC kernel reads.
"""
import torch

from . import lib
from .config import ModelConfig, VOC_STRIDES, VOC_DILATIONS, VOC_LRELU


def _fold(sd, prefix):
    g, v = sd[prefix + "weight_g"].float(), sd[prefix + "weight_v"].float()
    norm = v.reshape(v.shape[0], -1).norm(dim=1).reshape(v.shape[0], *([1] * (v.dim() - 1)))
    return g * v / norm


def _f(t, dev):
    return t.to(device=dev, dtype=torch.float32).contiguous()


class VocoderEngine:
    def __init__(self, sd, cfg: ModelConfig, device="cuda"):
        self.cfg = cfg
        self.dev = torch.device(device)
        dev = self.dev
        ch, hid = cfg.voc_channels, cfg.voc_kp_hidden
        self.ch, self.hid, self.nl = ch, hid, len(VOC_DILATIONS)
        self.conv_pre_w, self.conv_pre_b = _f(_fold(sd, "conv_pre."), dev), _f(sd["conv_pre.bias"], dev)
        self.conv_post_w, self.conv_post_b = _f(_fold(sd, "conv_post.1."), dev), _f(sd["conv_post.1.bias"], dev)
        self.blocks = []
        nk = ch * 2 * ch * 3           # kernel values per layer
        for b, s in enumerate(VOC_STRIDES):
            p = f"res_stack.{b}."
            kp = p + "kernel_predictor."
            blk = dict(stride=s)
            blk["convt_w"], blk["convt_b"] = _f(_fold(sd, p + "convt_pre.1."), dev), _f(sd[p + "convt_pre.1.bias"], dev)
            blk["in_w"], blk["in_b"] = _f(_fold(sd, kp + "input_conv.0."), dev), _f(sd[kp + "input_conv.0.bias"], dev)
            blk["res"] = [(_f(_fold(sd, kp + f"residual_convs.{r}.1."), dev), _f(sd[kp + f"residual_convs.{r}.1.bias"], dev),
                           _f(_fold(sd, kp + f"residual_convs.{r}.3."), dev), _f(sd[kp + f"residual_convs.{r}.3.bias"], dev))
                          for r in range(3)]
            # kernel_conv rows are ordered (layer, in, out, k) (vocoder.py:78-85); regroup to (layer, in, k, out) so the
            # LVC kernel reads 64 consecutive output channels; append the bias_conv rows (layer, out)
            kw = _fold(sd, kp + "kernel_conv.")                      # [nl*ch*2ch*3, hid, 3]
            kb = sd[kp + "kernel_conv.bias"].float()
            idx = torch.arange(self.nl * nk).reshape(self.nl, ch, 2 * ch, 3).permute(0, 1, 3, 2).reshape(-1)
            bw = _fold(sd, kp + "bias_conv.")                        # [nl*2ch, hid, 3]
            bb = sd[kp + "bias_conv.bias"].float()
            w_all = torch.cat([kw[idx], bw], dim=0)                  # [N, hid, 3]
            # error-compensated bf16 split (x = hi + lo): per tap the K axis is [Wh | Wh | Wl] against activations
            # [xh | xl | xh], i.e. xh*Wh + xl*Wh + xh*Wl ~ fp32-grade products on the bf16 tensor pipe
            wt = w_all.permute(0, 2, 1).contiguous()                 # [N, 3 taps, hid]
            wh = wt.to(torch.bfloat16)
            wl = (wt - wh.float()).to(torch.bfloat16)
            blk["kp_w"] = torch.cat([wh, wh, wl], dim=2).reshape(wt.shape[0], 3 * 3 * hid).to(dev).contiguous()
            blk["kp_b"] = _f(torch.cat([kb[idx], bb], dim=0), dev)
            blk["conv"] = [(_f(_fold(sd, p + f"conv_blocks.{d}.1."), dev), _f(sd[p + f"conv_blocks.{d}.1.bias"], dev))
                           for d in range(self.nl)]
            self.blocks.append(blk)
        self.kp_n = self.nl * nk + self.nl * 2 * ch
        self.nk = nk

    def inference(self, mel, z):
        """mel fp32 [100, S] (channel-major), z fp32 [64, S+10] -> waveform fp32 [256*S] in [-1, 1]."""
        cfg, dev, ch, hid = self.cfg, self.dev, self.ch, self.hid
        mel = _f(mel.reshape(cfg.voc_mel, -1), dev)
        S = mel.shape[1]
        F = S + 10
        c = torch.cat([mel, torch.full((cfg.voc_mel, 10), -11.5129, dtype=torch.float32, device=dev)], dim=1).contiguous()
        z = _f(z.reshape(cfg.voc_noise_dim, F), dev)
        x = torch.empty(ch, F, dtype=torch.float32, device=dev)
        lib.voc_conv1d(z, cfg.voc_noise_dim, F, self.conv_pre_w, self.conv_pre_b, ch, 7, x, reflect=True)
        L, hop = F, 1
        c1 = torch.empty(hid, F, dtype=torch.float32, device=dev)
        c2 = torch.empty(hid, F, dtype=torch.float32, device=dev)
        c3 = torch.empty(hid, F, dtype=torch.float32, device=dev)
        tok = torch.empty(F, 3 * hid, dtype=torch.bfloat16, device=dev)
        kern = torch.empty(F, self.kp_n, dtype=torch.float32, device=dev)
        for blk in self.blocks:
            s = blk["stride"]
            hop *= s
            xo = torch.empty(ch, L * s, dtype=torch.float32, device=dev)
            lib.voc_convt(x, ch, L, blk["convt_w"], blk["convt_b"], s, VOC_LRELU, xo)
            x, L = xo, L * s
            # kernel predictor (vocoder.py:66-93)
            lib.voc_conv1d(c, cfg.voc_mel, F, blk["in_w"], blk["in_b"], hid, 5, c1, lrelu_out=VOC_LRELU)
            cur, nxt = c1, c3
            for (w1, b1, w2, b2) in blk["res"]:
                lib.voc_conv1d(cur, hid, F, w1, b1, hid, 3, c2, lrelu_out=VOC_LRELU)
                lib.voc_conv1d(c2, hid, F, w2, b2, hid, 3, nxt, lrelu_out=VOC_LRELU, residual=cur)
                cur, nxt = nxt, cur
            lib.voc_to_tokens_bf16(cur, hid, F, tok, 3 * hid, split=True)
            lib.gemm(tok, blk["kp_w"], M=F, N=self.kp_n, K=3 * hid, taps=3, pad=1, bias=blk["kp_b"], out_f32=kern)
            y = torch.empty(ch, L, dtype=torch.float32, device=dev)
            for i, d in enumerate(VOC_DILATIONS):
                w, b = blk["conv"][i]
                lib.voc_conv1d(x, ch, L, w, b, ch, 3, y, dilation=d, lrelu_in=VOC_LRELU, lrelu_out=VOC_LRELU)
                lib.voc_lvc_gate(y, ch, L, hop, kern, self.kp_n, i * self.nk, kern, self.kp_n,
                                 self.nl * self.nk + i * 2 * ch, x)
        out = torch.empty(1, L, dtype=torch.float32, device=dev)
        lib.voc_conv1d(x, ch, L, self.conv_post_w, self.conv_post_b, 1, 7, out, reflect=True, lrelu_in=VOC_LRELU,
                       tanh_out=True)
        return out[0, : L - 256 * 10].clamp(-1, 1).contiguous()
