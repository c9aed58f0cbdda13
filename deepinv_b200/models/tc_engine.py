"""bf16 tensor-core execution of DRUNet / DnCNN (precision="bf16").

Activations stay NHWC bf16 in HBM between layers; every 3x3 convolution is one launch of the wgmma
implicit-GEMM kernel (csrc/conv_tc.cu) with ReLU / residual / U-Net-skip additions fused into its
epilogue; the network tail writes fp32 NCHW directly.  Weights are repacked once per parameter version
into the K-major (Cout, taps*Cin) bf16 layout the kernel's TMA descriptors expect.

Numerics: bf16 operands, fp32 accumulation — the same class as PyTorch's default GPU autocast; the fp32
path (precision="fp32") is the one that matches the reference to 1e-5.
"""
from __future__ import annotations

import torch

from .. import ops


def _pack3x3(w: torch.Tensor, cin_pad: int | None = None, rows_pad: int | None = None) -> torch.Tensor:
    """(Cout, Cin, 3, 3) -> (rows, 9*Cin_pad) bf16 with k = (ky*3+kx)*Cin_pad + c"""
    co, ci = w.shape[:2]
    cp = ci if cin_pad is None else cin_pad
    rp = co if rows_pad is None else rows_pad
    out = torch.zeros(rp, 3, 3, cp, dtype=torch.float32, device=w.device)
    out[:co, :, :, :ci] = w.detach().float().permute(0, 2, 3, 1)
    return out.reshape(rp, 9 * cp).to(torch.bfloat16).contiguous()


def _pack_down(w: torch.Tensor) -> torch.Tensor:
    """(Cout, Cin, 2, 2) -> (Cout, 4*Cin), k = (dy*2+dx)*Cin + c"""
    return w.detach().float().permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(torch.bfloat16).contiguous()


def _pack_up(w: torch.Tensor) -> torch.Tensor:
    """(Cin, Cout, 2, 2) -> (4*Cout, Cin), row = (dy*2+dx)*Cout + co"""
    return w.detach().float().permute(2, 3, 1, 0).reshape(-1, w.shape[0]).to(torch.bfloat16).contiguous()


def _version_key(model) -> tuple:
    return tuple((id(p), p.data_ptr(), p._version) for p in model.parameters())


def _pad64(c: int) -> int:
    return (c + 63) // 64 * 64


def _pack_head(w: torch.Tensor) -> torch.Tensor | None:
    """(64, Cin<=4, 3, 3) -> (64, 64) bf16 with k = (ky*3+kx)*Cin + c (zero padded): operand of the dedicated head
    kernel, which builds the im2col rows in shared memory from the NCHW fp32 input; None if the shape does not fit"""
    co, ci = w.shape[:2]
    if co != 64 or ci > 4:
        return None
    out = torch.zeros(64, 64, dtype=torch.float32, device=w.device)
    out[:, : 9 * ci] = w.detach().float().permute(0, 2, 3, 1).reshape(64, 9 * ci)
    return out.to(torch.bfloat16).contiguous()


class _DrunetPack:
    def __init__(self, m):
        nb = m.nb
        for conv in [m.m_head, m.m_tail]:
            pass
        self.key = _version_key(m)
        self.nc = [m.m_head.weight.shape[0], m.m_down1[nb].weight.shape[0], m.m_down2[nb].weight.shape[0],
                   m.m_down3[nb].weight.shape[0]]
        if any(c % 64 for c in self.nc):
            raise NotImplementedError("precision='bf16' needs channel counts that are multiples of 64 (tensor-core N/K tiles); "
                                      f"got nc={self.nc}; use precision='fp32'")
        self.cin0 = m.m_head.weight.shape[1]
        self.head64 = _pack_head(m.m_head.weight)
        self.head = None if self.head64 is not None else _pack3x3(m.m_head.weight, cin_pad=_pad64(self.cin0))
        self.tail = _pack3x3(m.m_tail.weight, rows_pad=16)
        self.cout = m.m_tail.weight.shape[0]
        rb = lambda blocks: [(_pack3x3(b.res[0].weight), _pack3x3(b.res[2].weight)) for b in blocks]
        self.down = [(rb(list(st)[:nb]), _pack_down(st[nb].weight)) for st in (m.m_down1, m.m_down2, m.m_down3)]
        self.body = rb(list(m.m_body))
        self.up = [(_pack_up(st[0].weight), rb(list(st)[1:])) for st in (m.m_up3, m.m_up2, m.m_up1)]


def _resblocks(t, blocks, skip=None):
    """x + conv(relu(conv(x))) chain; `skip` is added to the LAST block's output (the consumer's `x + x_k`)"""
    for i, (w0, w1) in enumerate(blocks):
        u = ops.conv3x3_bf16(t, w0, relu=True)
        t = ops.conv3x3_bf16(u, w1, res=t, res2=skip if i == len(blocks) - 1 else None)
    return t


def drunet_forward_bf16(model, x0: torch.Tensor) -> torch.Tensor:
    """x0: (B, C+1, H, W) fp32 (noise map already concatenated) -> (B, C_out, H, W) fp32"""
    pk = model._tc
    if pk is None or pk.key != _version_key(model):
        pk = model._tc = _DrunetPack(model)
    if pk.head64 is not None:
        x1 = ops.conv3x3_head_bf16(x0, pk.head64)
    else:
        x1 = ops.conv3x3_bf16(ops.nchw_to_nhwc_bf16(x0, _pad64(pk.cin0)), pk.head)
    skips = [x1]
    t = x1
    for blocks, wd in pk.down:
        t = _resblocks(t, blocks)
        t = ops.conv2x2_bf16(t, wd, wd.shape[0], up=False)
        skips.append(t)
    # skips = [x1, x2, x3, x4]; body output gets + x4, each up stage's output gets the next skip
    t = _resblocks(t, pk.body, skip=skips[3])
    for i, (wu, blocks) in enumerate(pk.up):
        t = ops.conv2x2_bf16(t, wu, wu.shape[0] // 4, up=True)
        t = _resblocks(t, blocks, skip=skips[2 - i])
    return ops.conv3x3_bf16_tail(t, pk.tail, pk.cout)


class _DncnnPack:
    def __init__(self, m):
        self.key = _version_key(m)
        nf = m.in_conv.weight.shape[0]
        if nf % 64:
            raise NotImplementedError("precision='bf16' needs nf to be a multiple of 64; use precision='fp32'")
        self.cin = m.in_conv.weight.shape[1]
        self.cout = m.out_conv.weight.shape[0]
        f32 = lambda b: None if b is None else b.detach().float().contiguous()
        self.first64 = _pack_head(m.in_conv.weight)
        self.first = (None if self.first64 is not None else _pack3x3(m.in_conv.weight, cin_pad=_pad64(self.cin)), f32(m.in_conv.bias))
        self.mid = [(_pack3x3(c.weight), f32(c.bias)) for c in m.conv_list]
        self.last = (_pack3x3(m.out_conv.weight, rows_pad=16), f32(m.out_conv.bias))


def dncnn_forward_bf16(model, x: torch.Tensor) -> torch.Tensor:
    pk = model._tc
    if pk is None or pk.key != _version_key(model):
        pk = model._tc = _DncnnPack(model)
    if pk.first64 is not None:
        t = ops.conv3x3_head_bf16(x, pk.first64, bias=pk.first[1], relu=True)
    else:
        t = ops.conv3x3_bf16(ops.nchw_to_nhwc_bf16(x, _pad64(pk.cin)), pk.first[0], bias=pk.first[1], relu=True)
    for w, b in pk.mid:
        t = ops.conv3x3_bf16(t, w, bias=b, relu=True)
    return ops.conv3x3_bf16_tail(t, pk.last[0], pk.cout, bias=pk.last[1], add=x)


# ---------------------------------------------------------------------------------------------------------
# precision="tc32" / "tc32h": fp32-grade tensor-core execution (split operands, csrc/conv_tc32.cu)
#   tc32  : 3 x TF32, fp32-word "split16" activations, no range restriction
#   tc32h : 3 x FP16, fp16-word "split32h" activations (twice the channels per MMA, half the bytes); activations must stay
#           below 65504 in magnitude — beyond that the sticky overflow flag is raised and the output is NaN
# ---------------------------------------------------------------------------------------------------------
def _rna_tf32(w: torch.Tensor) -> torch.Tensor:
    """round to the nearest tf32 value (10-bit mantissa, ties away from zero: the device's cvt.rna.tf32.f32)"""
    u = w.contiguous().view(torch.int32)
    return torch.bitwise_and(u + 0x1000, -0x2000).view(torch.float32)


def _fmt(precision: str) -> int:
    return {"tc32": 0, "tc32h": 1}[precision]


def _pack_tc32(wk: torch.Tensor, fmt: int = 0) -> torch.Tensor:
    """K-major GEMM matrix (rows, K) fp32, rows % 64 == 0 -> (2*rows, K): per 64 rows [hi (64); lo (64)]
    fmt 0: tf32-rounded fp32 words;  fmt 1: fp16 words, lo scaled by 2^11"""
    wk = wk.detach().float().contiguous()
    rows, K = wk.shape
    if fmt == 0:
        hi = _rna_tf32(wk)
        lo = _rna_tf32(wk - hi)
    else:
        hi = wk.to(torch.float16)
        lo = ((wk - hi.float()) * 2048.0).to(torch.float16)
    return torch.cat([hi.view(rows // 64, 64, K), lo.view(rows // 64, 64, K)], dim=1).reshape(2 * rows, K).contiguous()


def _pack3x3_tc32(w, fmt: int = 0):   # (Cout, Cin, 3, 3) -> k = (ky*3+kx)*Cin + c
    return _pack_tc32(w.detach().float().permute(0, 2, 3, 1).reshape(w.shape[0], -1), fmt)


def _pack3x3_slab_tc32(w, fmt: int = 0):
    """(Cout, Cin, 3, 3) -> the halo kernel's K order: column ((c/CH * 5 + tap/2) * 2 + tap%2) * CH + c%CH, tap 9 = zeros"""
    ch = 32 if fmt == 1 else 16
    w = w.detach().float()
    co, ci = w.shape[:2]
    out = torch.zeros(co, ci // ch, 5, 2, ch, dtype=torch.float32, device=w.device)
    for tap in range(9):
        out[:, :, tap // 2, tap % 2, :] = w[:, :, tap // 3, tap % 3].reshape(co, ci // ch, ch)
    return _pack_tc32(out.reshape(co, 10 * ci), fmt)


def _pack_down_tc32(w, fmt: int = 0):  # (Cout, Cin, 2, 2) -> k = (dy*2+dx)*Cin + c
    return _pack_tc32(w.detach().float().permute(0, 2, 3, 1).reshape(w.shape[0], -1), fmt)


def _pack_up_tc32(w, fmt: int = 0):    # (Cin, Cout, 2, 2) -> row = (dy*2+dx)*Cout + co
    return _pack_tc32(w.detach().float().permute(2, 3, 1, 0).reshape(-1, w.shape[0]), fmt)


class _DrunetPack32:
    def __init__(self, m, fmt):
        nb = m.nb
        self.key = (_version_key(m), fmt)
        self.fmt = fmt
        self.nc = [m.m_head.weight.shape[0], m.m_down1[nb].weight.shape[0], m.m_down2[nb].weight.shape[0],
                   m.m_down3[nb].weight.shape[0]]
        if any(c % 64 for c in self.nc) or m.m_head.weight.shape[1] > 4 or m.m_tail.weight.shape[0] > 4 or self.nc[0] > 128:
            raise NotImplementedError("precision='tc32' / 'tc32h' need channel counts that are multiples of 64 (tensor-core N/K tiles), "
                                      f"at most 4 image channels and nc[0] <= 128; got nc={self.nc}; use precision='fp32'")
        self.head = m.m_head.weight.detach().float().contiguous()
        self.tail = m.m_tail.weight.detach().float().contiguous()
        self.flag = torch.zeros(1, dtype=torch.int32, device=self.head.device)
        rb = lambda blocks: [(_pack3x3_slab_tc32(b.res[0].weight, fmt), _pack3x3_slab_tc32(b.res[2].weight, fmt), b.res[0].weight.shape[0])
                             for b in blocks]
        self.down = [(rb(list(st)[:nb]), _pack_down_tc32(st[nb].weight, fmt), st[nb].weight.shape[0]) for st in (m.m_down1, m.m_down2, m.m_down3)]
        self.body = rb(list(m.m_body))
        self.up = [(_pack_up_tc32(st[0].weight, fmt), st[0].weight.shape[1], rb(list(st)[1:])) for st in (m.m_up3, m.m_up2, m.m_up1)]


def _resblocks32(t, blocks, flag, skip=None):
    for i, (w0, w1, c) in enumerate(blocks):
        u = ops.conv_tc32_slab(t, w0, c, relu=True, flag=flag)
        t = ops.conv_tc32_slab(u, w1, c, res=t, res2=skip if i == len(blocks) - 1 else None, flag=flag)
    return t


def drunet_forward_tc32(model, x0: torch.Tensor) -> torch.Tensor:
    """x0: (B, C+1, H, W) fp32 (noise map already concatenated) -> (B, C_out, H, W) fp32; same dataflow as the bf16 engine"""
    fmt = _fmt(model.precision)
    pk = model._tc32
    if pk is None or pk.key != (_version_key(model), fmt):
        pk = model._tc32 = _DrunetPack32(model, fmt)
    f = pk.flag if fmt == 1 else None
    if f is not None:
        f.zero_()   # the flag is per call: an out-of-range input poisons its own output, not the model
    x1 = ops.conv_tc32_head(x0, pk.head, fmt=fmt, flag=f)
    skips = [x1]
    t = x1
    for blocks, wd, cd in pk.down:
        t = _resblocks32(t, blocks, f)
        t = ops.conv_tc32(t, wd, cd, kind=1, flag=f)
        skips.append(t)
    t = _resblocks32(t, pk.body, f, skip=skips[3])
    for i, (wu, cu, blocks) in enumerate(pk.up):
        t = ops.conv_tc32(t, wu, cu, kind=2, flag=f)
        t = _resblocks32(t, blocks, f, skip=skips[2 - i])
    return ops.conv_tc32_tail(t, pk.tail, flag=f)


# ---- DRUNet(dim=3): the same dataflow on NDHWC split volumes, every layer on the per-tap kernel (csrc/conv_tc32.cu, D3) ----
def _pack3x3x3_tc32(w, fmt: int = 0):   # (Cout, Cin, 3, 3, 3) -> k = ((kz*3+ky)*3+kx)*Cin + c
    return _pack_tc32(w.detach().float().permute(0, 2, 3, 4, 1).reshape(w.shape[0], -1), fmt)


def _pack_down3d_tc32(w, fmt: int = 0):  # (Cout, Cin, 2, 2, 2) -> k = (dz*4+dy*2+dx)*Cin + c
    return _pack_tc32(w.detach().float().permute(0, 2, 3, 4, 1).reshape(w.shape[0], -1), fmt)


def _pack_up3d_tc32(w, fmt: int = 0):    # (Cin, Cout, 2, 2, 2) -> row = (dz*4+dy*2+dx)*Cout + co
    return _pack_tc32(w.detach().float().permute(2, 3, 4, 1, 0).reshape(-1, w.shape[0]), fmt)


class _Drunet3dPack32(_DrunetPack32):
    def __init__(self, m, fmt):
        from .drunet import body_blocks

        nb = m.nb
        self.key = (_version_key(m), fmt)
        self.fmt = fmt
        self.nc = [m.m_head.weight.shape[0], m.m_down1[nb].weight.shape[0], m.m_down2[nb].weight.shape[0],
                   m.m_down3[nb].weight.shape[0]]
        if any(c % 64 for c in self.nc) or m.m_head.weight.shape[1] > 4 or m.m_tail.weight.shape[0] > 4 or self.nc[0] > 128:
            raise NotImplementedError("precision='tc32' / 'tc32h' need channel counts that are multiples of 64 (tensor-core N/K tiles), "
                                      f"at most 4 image channels and nc[0] <= 128; got nc={self.nc}; use precision='fp32'")
        self.head = m.m_head.weight.detach().float().contiguous()
        self.tail = m.m_tail.weight.detach().float().contiguous()
        self.flag = torch.zeros(1, dtype=torch.int32, device=self.head.device)
        rb = lambda blocks: [(_pack3x3x3_tc32(b.res[0].weight, fmt), _pack3x3x3_tc32(b.res[2].weight, fmt), b.res[0].weight.shape[0])
                             for b in blocks]
        self.down = [(rb(list(st)[:nb]), _pack_down3d_tc32(st[nb].weight, fmt), st[nb].weight.shape[0]) for st in (m.m_down1, m.m_down2, m.m_down3)]
        self.body = rb(body_blocks(m))
        self.up = [(_pack_up3d_tc32(st[0].weight, fmt), st[0].weight.shape[1], rb(list(st)[1:])) for st in (m.m_up3, m.m_up2, m.m_up1)]


def _resblocks3d32(t, blocks, flag, skip=None):
    for i, (w0, w1, c) in enumerate(blocks):
        u = ops.conv3d_tc32(t, w0, c, relu=True, flag=flag)
        t = ops.conv3d_tc32(u, w1, c, res=t, res2=skip if i == len(blocks) - 1 else None, flag=flag)
    return t


def drunet3d_forward_tc32(model, x0: torch.Tensor) -> torch.Tensor:
    """x0: (B, C+1, D, H, W) fp32 (noise map already concatenated) -> (B, C_out, D, H, W) fp32; the dataflow of drunet_forward_tc32"""
    fmt = _fmt(model.precision)
    pk = model._tc32
    if not isinstance(pk, _Drunet3dPack32) or pk.key != (_version_key(model), fmt):
        pk = model._tc32 = _Drunet3dPack32(model, fmt)
    f = pk.flag if fmt == 1 else None
    if f is not None:
        f.zero_()   # the flag is per call: an out-of-range input poisons its own output, not the model
    x1 = ops.conv3d_tc32_head(x0, pk.head, fmt=fmt, flag=f)
    skips = [x1]
    t = x1
    for blocks, wd, cd in pk.down:
        t = _resblocks3d32(t, blocks, f)
        t = ops.conv3d_tc32(t, wd, cd, kind=1, flag=f)
        skips.append(t)
    t = _resblocks3d32(t, pk.body, f, skip=skips[3])
    for i, (wu, cu, blocks) in enumerate(pk.up):
        t = ops.conv3d_tc32(t, wu, cu, kind=2, flag=f)
        t = _resblocks3d32(t, blocks, f, skip=skips[2 - i])
    return ops.conv3d_tc32_tail(t, pk.tail, flag=f)


class _DncnnPack32:
    def __init__(self, m, fmt):
        self.key = (_version_key(m), fmt)
        self.fmt = fmt
        nf = m.in_conv.weight.shape[0]
        if nf % 64 or nf > 128 or m.in_conv.weight.shape[1] > 4 or m.out_conv.weight.shape[0] > 4:
            raise NotImplementedError("precision='tc32' / 'tc32h' need nf in {64, 128} and at most 4 image channels; use precision='fp32'")
        f32 = lambda b: None if b is None else b.detach().float().contiguous()
        self.nf = nf
        self.first = (m.in_conv.weight.detach().float().contiguous(), f32(m.in_conv.bias))
        self.mid = [(_pack3x3_slab_tc32(c.weight, fmt), f32(c.bias)) for c in m.conv_list]
        self.last = (m.out_conv.weight.detach().float().contiguous(), f32(m.out_conv.bias))
        self.flag = torch.zeros(1, dtype=torch.int32, device=self.first[0].device)


def dncnn_forward_tc32(model, x: torch.Tensor) -> torch.Tensor:
    fmt = _fmt(model.precision)
    pk = model._tc32
    if pk is None or pk.key != (_version_key(model), fmt):
        pk = model._tc32 = _DncnnPack32(model, fmt)
    f = pk.flag if fmt == 1 else None
    if f is not None:
        f.zero_()
    t = ops.conv_tc32_head(x, pk.first[0], bias=pk.first[1], relu=True, fmt=fmt, flag=f)
    for w, b in pk.mid:
        t = ops.conv_tc32_slab(t, w, pk.nf, bias=b, relu=True, flag=f)
    return ops.conv_tc32_tail(t, pk.last[0], bias=pk.last[1], add=x, flag=f)


def tc_overflow(model) -> bool:
    """True if an activation of the LAST precision='tc32h' forward left the fp16 range (that call's output is NaN, every kernel
    after the overflow having seen the raised flag); host-synchronising read of the device flag, which each forward clears"""
    pk = getattr(model, "_tc32", None)
    return bool(pk is not None and pk.fmt == 1 and int(pk.flag.item()) != 0)
