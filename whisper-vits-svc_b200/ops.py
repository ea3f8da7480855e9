"""Single-operator entry points of the C ABI on torch CUDA tensors (unit tests / profiling).
The same kernels the stage pipelines launch; no fallback."""
from __future__ import annotations

import torch

from . import _lib, pack


def _c(t):
    assert t.is_cuda, "operators run on CUDA tensors only"
    return t.float().contiguous()


def conv1d(x, weight, bias=None, stride=1, padding=0, dilation=1, act=0):
    """weight in torch layout [Cout,Cin,K]; packed here (host) then run on the device."""
    x = _c(x)
    B, Cin, Tin = x.shape
    Cout, _, K = weight.shape
    wp = pack.pack_conv(weight.detach().cpu().float()).to(x.device)
    b = _c(bias) if bias is not None else None
    Tout = (Tin + 2 * padding - dilation * (K - 1) - 1) // stride + 1
    y = torch.empty(B, Cout, Tout, device=x.device)
    _lib.call("op_conv1d", x.data_ptr(), wp.data_ptr(), b.data_ptr() if b is not None else None,
              y.data_ptr(), B, Cin, Cout, Tin, K, stride, dilation, padding, act, device=x.device)
    return y


def snake_alias(x, alpha, beta, fu, fd):
    x = _c(x)
    B, C, L = x.shape
    ea = _c(torch.exp(alpha.float().cpu()).to(x.device))
    ib = _c((1.0 / (torch.exp(beta.float().cpu()) + 1e-9)).to(x.device))
    fu, fd = _c(fu.reshape(-1).to(x.device)), _c(fd.reshape(-1).to(x.device))
    y = torch.empty_like(x)
    _lib.call("op_snake_alias", x.data_ptr(), y.data_ptr(), ea.data_ptr(), ib.data_ptr(),
              fu.data_ptr(), fd.data_ptr(), B, C, L, device=x.device)
    return y


def layernorm_c(x, r, gamma, beta, eps=1e-5):
    x = _c(x)
    B, C, T = x.shape
    gamma, beta = _c(gamma), _c(beta)
    stride = C if gamma.dim() == 2 else 0
    r_ = _c(r) if r is not None else None
    y = torch.empty_like(x)
    _lib.call("op_layernorm_c", x.data_ptr(), r_.data_ptr() if r_ is not None else None,
              gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), B, C, T, stride, eps, device=x.device)
    return y


def rel_attention(qkv, emb_k, emb_v, lengths, heads=2, window=4, tc=False):
    qkv = _c(qkv)
    B, H3, T = qkv.shape
    H = H3 // 3
    ek, ev = _c(emb_k.reshape(2 * window + 1, -1)), _c(emb_v.reshape(2 * window + 1, -1))
    lengths = lengths.to(qkv.device, torch.int64).contiguous()
    out = torch.empty(B, H, T, device=qkv.device)
    if tc:
        scratch = torch.empty(int(_lib.load().svcb_op_rel_attention_tc_scratch_bytes(B, heads, T)), dtype=torch.uint8,
                              device=qkv.device)
        _lib.call("op_rel_attention_tc", qkv.data_ptr(), ek.data_ptr(), ev.data_ptr(), lengths.data_ptr(), out.data_ptr(),
                  B, H, heads, window, T, scratch.data_ptr(), scratch.numel(), device=qkv.device)
        return out
    _lib.call("op_rel_attention", qkv.data_ptr(), ek.data_ptr(), ev.data_ptr(), lengths.data_ptr(),
              out.data_ptr(), B, H, heads, window, T, device=qkv.device)
    return out


def amp_conv_tc(x, alpha, beta, fu, fd, weight, bias, dilation=1, res=None, nsplit=3, acc=None, out_div=0.0):
    """SnakeAlias -> Conv1d(C->C, K, dilation, 'same') + bias (+res) on the tensor cores.  acc: a stage sum
    [B, C, L] that the result is added to (in a copy), then divided by out_div when it is not 0."""
    x = _c(x)
    B, C, L = x.shape
    K = weight.shape[-1]
    ea = _c(torch.exp(alpha.float().cpu()).to(x.device))
    ib = _c((1.0 / (torch.exp(beta.float().cpu()) + 1e-9)).to(x.device))
    fu, fd = _c(fu.reshape(-1).to(x.device)), _c(fd.reshape(-1).to(x.device))
    wtc = pack.pack_conv_tc(weight.detach().cpu().float()).to(x.device)
    b = _c(bias)
    r = _c(res) if res is not None else None
    y = _c(acc).clone() if acc is not None else torch.empty_like(x)
    scratch = torch.empty(int(_lib.load().svcb_op_amp_conv_tc_scratch_bytes(B, C, L)), dtype=torch.uint8, device=x.device)
    _lib.call("op_amp_conv_tc", x.data_ptr(), y.data_ptr(), r.data_ptr() if r is not None else None,
              ea.data_ptr(), ib.data_ptr(), fu.data_ptr(), fd.data_ptr(),
              wtc.data_ptr(), b.data_ptr(), B, C, L, K, dilation, nsplit, int(acc is not None), float(out_div),
              scratch.data_ptr(), scratch.numel(), device=x.device)
    return y


def amp_s2d_link(x, alpha_in, beta_in, fu, fd, weight, bias, dilation=1, res=None, alpha_out=None, beta_out=None,
                 out_dilation=1):
    """SnakeAlias_in -> Conv1d(C->C, K, dilation, 'same') + bias (+res) [-> SnakeAlias_out] in space-to-depth
    form (C = 20 / 10), on the input fold pack.s2d_fold picks.  Returns (y, y_act): the fp32 result and, when
    alpha_out is given, the next link's operand image decoded back to fp32 (written folded for a next link of
    dilation out_dilation when that is > 1)."""
    x = _c(x)
    B, C, L = x.shape
    K = weight.shape[-1]
    r = pack.s2d_factor(C)

    def snake_params(a, b):
        return (_c(torch.exp(a.float().cpu()).to(x.device)), _c((1.0 / (torch.exp(b.float().cpu()) + 1e-9)).to(x.device)))

    ea_i, ib_i = snake_params(alpha_in, beta_in)
    ea_o, ib_o = snake_params(alpha_out, beta_out) if alpha_out is not None else (None, None)
    fu, fd = _c(fu.reshape(-1).to(x.device)), _c(fd.reshape(-1).to(x.device))
    w = pack.pack_conv_s2d_link(weight.detach().cpu().float(), dilation, r).to(x.device)
    b = _c(bias)
    rs = _c(res) if res is not None else None
    y = torch.empty_like(x)
    y_act = torch.empty_like(x) if alpha_out is not None else None
    scratch = torch.empty(int(_lib.load().svcb_op_amp_s2d_link_scratch_bytes(B, C, L)), dtype=torch.uint8, device=x.device)
    _lib.call("op_amp_s2d_link", x.data_ptr(), y.data_ptr(), rs.data_ptr() if rs is not None else None,
              y_act.data_ptr() if y_act is not None else None, ea_i.data_ptr(), ib_i.data_ptr(),
              ea_o.data_ptr() if ea_o is not None else None, ib_o.data_ptr() if ib_o is not None else None,
              fu.data_ptr(), fd.data_ptr(), w.data_ptr(), b.data_ptr(), B, C, L, K, dilation, out_dilation,
              scratch.data_ptr(), scratch.numel(), device=x.device)
    return y, y_act


def amp_s2d_link_ragged(x, lens, alpha_in, beta_in, fu, fd, weight, bias, dilation=1, res=None, alpha_out=None,
                        beta_out=None, out_dilation=1):
    """amp_s2d_link over a ragged batch: item b is x[b, :, :lens[b]] (each a multiple of 8 and of 160 / C).
    Returns (y, y_act, out_hi, out_lo): y and y_act as amp_s2d_link's, zero past each item's end, and the
    output S2D image as written (folded when out_dilation > 1), bf16 [B, 20, Rp, 8] hi and lo (None without
    alpha_out)."""
    x = _c(x)
    B, C, L = x.shape
    K = weight.shape[-1]
    r = pack.s2d_factor(C)

    def snake_params(a, b):
        return (_c(torch.exp(a.float().cpu()).to(x.device)), _c((1.0 / (torch.exp(b.float().cpu()) + 1e-9)).to(x.device)))

    ea_i, ib_i = snake_params(alpha_in, beta_in)
    ea_o, ib_o = snake_params(alpha_out, beta_out) if alpha_out is not None else (None, None)
    fu, fd = _c(fu.reshape(-1).to(x.device)), _c(fd.reshape(-1).to(x.device))
    w = pack.pack_conv_s2d_link(weight.detach().cpu().float(), dilation, r).to(x.device)
    b = _c(bias)
    rs = _c(res) if res is not None else None
    ln = torch.as_tensor(lens, dtype=torch.int32).cpu().contiguous()
    y = torch.zeros_like(x)
    y_act = torch.zeros_like(x) if alpha_out is not None else None
    nbytes = int(_lib.load().svcb_op_amp_s2d_link_scratch_bytes(B, C, L))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    _lib.call("op_amp_s2d_link_ragged", x.data_ptr(), y.data_ptr(), rs.data_ptr() if rs is not None else None,
              y_act.data_ptr() if y_act is not None else None, ea_i.data_ptr(), ib_i.data_ptr(),
              ea_o.data_ptr() if ea_o is not None else None, ib_o.data_ptr() if ib_o is not None else None,
              fu.data_ptr(), fd.data_ptr(), w.data_ptr(), b.data_ptr(), ln.data_ptr(), B, C, L, K, dilation, out_dilation,
              scratch.data_ptr(), scratch.numel(), device=x.device)
    if alpha_out is None:
        return y, y_act, None, None
    img = (nbytes - 512) // 4
    S = 128 - 2 * (1 if r >= 8 else 2)                   # useful rows per tile (amp_s2d.cu: s2d_rows)
    rows = -(-(L // r) // S) * S + 160

    def image(i):
        return scratch[i * img:i * img + B * 20 * rows * 16].view(torch.bfloat16).view(B, 20, rows, 8)

    return y, y_act, image(2), image(3)


def conv_tc(x, weight, bias=None, dilation=1, res=None, lengths=None, nsplit=3, flags=0, act=0):
    """Stride-1 'same' Conv1d on the tensor cores; weight in torch layout [Cout,Cin,K]."""
    x = _c(x)
    B, Cin, T = x.shape
    Cout, _, K = weight.shape
    wtc = pack.pack_conv_tc_general(weight.detach().cpu().float()).to(x.device)
    b = _c(bias) if bias is not None else None
    r = _c(res) if res is not None else None
    ln = lengths.to(x.device, torch.int64).contiguous() if lengths is not None else None
    cout_real = Cout // 2 if (flags & 4) else Cout
    y = torch.zeros(B, cout_real, T, device=x.device)
    _lib.call("op_conv_tc", x.data_ptr(), wtc.data_ptr(), b.data_ptr() if b is not None else None,
              y.data_ptr(), r.data_ptr() if r is not None else None,
              ln.data_ptr() if ln is not None else None, B, Cin, Cout, T, K, dilation,
              nsplit, flags, act, device=x.device)
    return y
