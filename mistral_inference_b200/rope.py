"""RoPE table (mirror of mistral_inference/rope.py:6-10).

The table is built on the CPU in fp32 exactly as the reference does (transformer.py:108-120 builds it on
the default device, then moves it) and uploaded, so the kernels multiply by the very same cos/sin bits
instead of calling sincosf on the device (SURVEY.md Appendix A-3).  The rotation itself
(rope.py:13-23) is the epilogue of the fused QKV kernel (csrc/epilogue.cuh, EPI_QKV_ROPE).
"""
import torch


def precompute_freqs_cis(dim: int, end: int, theta: float) -> torch.Tensor:
    """complex64 [end, dim/2]: polar(1, t * theta^(-2i/dim))."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2)[: (dim // 2)].float() / dim))
    t = torch.arange(end, device=freqs.device)
    freqs = torch.outer(t, freqs).float()
    return torch.polar(torch.ones_like(freqs), freqs)


def precompute_freqs_cis_2d(dim: int, height: int, width: int, theta: float) -> torch.Tensor:
    """complex64 [height, width, dim/2] (rope.py:26-51): the first dim/4 frequencies rotate by the patch row, the last dim/4 by
    the column.  The vision encoder flattens it to [height * width, dim/2] and indexes it with row * width + col."""
    freqs = 1.0 / (theta ** (torch.arange(0, dim, 2).float() / dim))
    h = torch.arange(height, device=freqs.device)
    w = torch.arange(width, device=freqs.device)
    freqs_h = torch.outer(h, freqs[::2]).float()
    freqs_w = torch.outer(w, freqs[1::2]).float()
    freqs_2d = torch.cat([freqs_h[:, None, :].repeat(1, width, 1), freqs_w[None, :, :].repeat(height, 1, 1)], dim=-1)
    return torch.polar(torch.ones_like(freqs_2d), freqs_2d)
