"""Cosine-similarity GEMM of the appearance branch on the wgmma conv kernel (SURVEY.md section 8f row 3).

``matching.embedding_distance`` / ``cal_cosine_distance`` (tracker/matching.py:84-103, 165-178) compute
``normalize(tracks) @ normalize(detections).T`` -- an N x 512 x M contraction, the one genuine tensor-core GEMM on the association
side.  It runs here as a 1 x 1 "convolution" of csrc/b2t_conv.cu: the N track features are the pixels, the M detection features the
output channels.  To keep the reference's float64-level results on fp16 tensor cores each unit vector is split into two fp16 terms,
x = hi + lo with hi = fp16(x), lo = fp16(x - hi), and ONE GEMM over the concatenated K axis
    [a_hi | a_hi | a_lo] . [b_hi | b_lo | b_hi]^T  =  a_hi.b_hi + a_hi.b_lo + a_lo.b_hi
recovers the product to ~2^-22 (fp16 x fp16 products are exact in the fp32 accumulator; the dropped lo.lo term is 2^-22 relative).
"""
import torch

from . import _lib as L
from .conv import ConvPlan


class CosineGemm:
    def __init__(self, device="cuda:0", dim=512, n_max=512, m_max=512):
        if not torch.cuda.is_available():
            raise L.B2TError("CosineGemm needs a CUDA device: there is no CPU fallback")
        self.dev = torch.device(device)
        self.dim = self.n_max = self.m_max = 0
        self._alloc(dim, n_max, m_max)

    def _alloc(self, dim, n_max, m_max):
        kd = (dim + 63) // 64 * 64                         # the kernel's K chunk is 64 channels
        n_max, m_max = (n_max + 127) // 128 * 128, (m_max + 63) // 64 * 64
        self.dim, self.kd, self.n_max, self.m_max = dim, kd, n_max, m_max
        self.a = torch.zeros((1, 1, n_max, 3 * kd), dtype=torch.float16, device=self.dev)       # NHWC "image": n_max pixels x 3 kd channels
        self.w = torch.zeros((m_max, 3 * kd), dtype=torch.float16, device=self.dev)             # [cout rows][K]
        self.bias = torch.zeros(m_max, dtype=torch.float32, device=self.dev)
        self.out = torch.zeros((1, 1, n_max, m_max), dtype=torch.float32, device=self.dev)
        self.plan = ConvPlan(self.a, self.w, self.bias, self.out, 1, 1, n_max, 3 * kd, 0, m_max, 1, 1, 0, act=False, out_f32=True)

    @staticmethod
    def _split(x):
        hi = x.to(torch.float16)
        lo = (x - hi.to(x.dtype)).to(torch.float16)
        return hi, lo

    def cosine_similarity(self, tracks, dets):
        """tracks (N, dim), dets (M, dim): CUDA tensors (any float dtype) -> (N, M) float32 cosine similarities on the device."""
        n, m = tracks.shape[0], dets.shape[0]
        if tracks.shape[1] != self.dim or n > self.n_max or m > self.m_max:
            self._alloc(tracks.shape[1], max(n, self.n_max), max(m, self.m_max))
        a = tracks.to(self.dev, torch.float64)
        b = dets.to(self.dev, torch.float64)
        a = a / a.norm(dim=1, keepdim=True)
        b = b / b.norm(dim=1, keepdim=True)
        a_hi, a_lo = self._split(a)
        b_hi, b_lo = self._split(b)
        kd, d = self.kd, self.dim
        av, wv = self.a[0, 0], self.w
        av[:n, 0:d], av[:n, kd:kd + d], av[:n, 2 * kd:2 * kd + d] = a_hi, a_hi, a_lo
        wv[:m, 0:d], wv[:m, kd:kd + d], wv[:m, 2 * kd:2 * kd + d] = b_hi, b_lo, b_hi
        self.plan.run()
        return self.out[0, 0, :n, :m]
