"""Host side of the wgmma conv kernel (csrc/b2t_conv.cu): weight packing and plan objects.

``pack_conv_weight`` turns a (BN-folded) ``[Cout, Cin, KH, KW]`` fp32 weight into the K-major
``[Cout_rows, KH, KW, Cin_pad]`` bf16 layout the B-operand tensor map reads.  ``ConvPlan`` owns the
TMA descriptors for one layer; buffers are NHWC bf16 / fp16 torch tensors (possibly wider than the slice used).
"""
import ctypes as C

import torch

from . import _lib as L


def pack_conv_weight(w, cin_pad=None, dtype=torch.bfloat16):
    """w: (Cout, Cin, KH, KW) float -> (Cout_rows, KH*KW*Cin_pad) bf16 / fp16 contiguous, rows padded to 16."""
    cout, cin, kh, kw = w.shape
    cin_pad = cin_pad or (cin + 15) // 16 * 16
    rows = (cout + 15) // 16 * 16
    out = torch.zeros((rows, kh, kw, cin_pad), dtype=torch.float32, device=w.device)
    out[:cout, :, :, :cin] = w.permute(0, 2, 3, 1)
    return out.reshape(rows, kh * kw * cin_pad).to(dtype).contiguous()


def pack_conv_weight_rowpack(w, dtype=torch.bfloat16):
    """Row-packed stem layout (b2t_conv_desc.rowpack): w (Cout, Cin <= 16, 3, 3) -> (Cout_rows, 3 * 64) bf16 with
    k = kh * 64 + kw * 16 + c; columns 48..63 of every kernel row (the dummy fourth pixel) stay zero."""
    cout, cin, kh, kw = w.shape
    assert kh == 3 and kw == 3 and cin <= 16
    rows = (cout + 15) // 16 * 16
    out = torch.zeros((rows, 3, 4, 16), dtype=torch.float32, device=w.device)
    out[:cout, :, :3, :cin] = w.permute(0, 2, 3, 1)
    return out.reshape(rows, 192).to(dtype).contiguous()


class ConvPlan:
    def __init__(self, x, w_packed, bias, y, n, h, w, cin, in_coff, cout, k, stride, out_coff, act=True, out_f32=False,
                 block_n=0, tile_w=0, stages=0, in_row_pixels=0, rowpack=False, x_pixel0=0, halo=False, mt=1, splits=1, halo_bufs=0, producers=0, tps=0, out_bufs=0, kpair=0):
        """x: NHWC bf16 buffer (n, h, w, in_pitch) -- or (n, h, in_row_pixels, in_pitch) with x_pixel0 = first pixel the plan
        addresses in a row; y: NHWC buffer (n, ho, wo, out_pitch) bf16 or fp32."""
        self.lib = L.load()
        assert x.dtype in (torch.bfloat16, torch.float16) and x.is_contiguous() and y.is_contiguous()
        assert w_packed.dtype == x.dtype and bias.dtype == torch.float32 and (out_f32 or y.dtype == x.dtype)
        self.keep = (x, w_packed, bias, y)
        self.geom = dict(n=n, h=h, w=w, cin=cin, cout=cout, k=k, stride=stride, out_f32=bool(out_f32), rowpack=bool(rowpack))
        d = L.ConvDesc(x=x.data_ptr() + x_pixel0 * x.shape[-1] * 2, w_packed=w_packed.data_ptr(), bias=bias.data_ptr(), y=y.data_ptr(), n=n, h=h, w=w,
                       cin=cin, in_pitch=x.shape[-1], in_coff=in_coff, cout=cout, cout_rows=w_packed.shape[0], kh=k, kw=k,
                       stride=stride, out_pitch=y.shape[-1], out_coff=out_coff, act=int(act), out_f32=int(out_f32),
                       block_n=block_n, tile_w=tile_w, stages=stages, in_row_pixels=in_row_pixels, rowpack=int(rowpack), io_dtype=L.act_dtype_code(x.dtype),
                       halo=int(halo), halo_bufs=int(halo_bufs), tps=int(tps), kpair=int(kpair), out_bufs=int(out_bufs), mt=int(mt), producers=int(producers), splits=int(splits))
        self.handle = C.c_void_p()
        rc = self.lib.b2t_conv_plan_create(C.byref(d), C.byref(self.handle))
        if rc != 0:
            raise L.B2TError("b2t_conv_plan_create: %s" % (self.lib.b2t_conv_last_error() or b"").decode())
        self.flops = self.lib.b2t_conv_plan_flops(self.handle)
        info = (C.c_int * 17)()
        self.lib.b2t_conv_plan_info(self.handle, info, 17)
        self.info = dict(zip(("grid", "threads", "smem", "bn", "stages", "mt", "splits", "halo", "halo_bufs", "tiles_m", "tiles_n", "acc_regs", "producers", "tps", "b_res", "out_bufs", "kpair"), list(info)))

    def run(self, stream=None):
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream if stream is None else stream)
        rc = self.lib.b2t_conv_run(self.handle, s)
        if rc != 0:
            raise L.B2TError("b2t_conv_run: %s" % (self.lib.b2t_conv_last_error() or b"").decode())

    def __del__(self):
        try:
            if self.handle:
                self.lib.b2t_conv_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass
