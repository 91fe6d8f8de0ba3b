"""Torch restatement of satb_sampler_step (csrc/sampler.cu; the algebra of SatbSamplerStep in include/satb200.h),
used on the CPU to drive the native step path of inference/sampling.py without a GPU, and on the GPU as the
element-by-element reference of the kernel.  ``p`` is the dict ``sampling._launch_step`` receives."""
import torch


def sampler_step_ref(p, dtype=None):
    """Evaluates in ``dtype`` (default: the state's); the blend rounds as the kernel does, in the state's dtype."""
    dtype = dtype or p["x"].dtype
    f = lambda t: None if t is None else t.to(dtype)
    x, y = f(p["x"]), f(p["y"])
    den = p["c_out"] * y + p["c_skip"] * x
    if p["mask"] is not None:
        L = p["L"]
        keep = p["mask"].to(torch.float32) <= torch.tensor(p["blend_thr"], dtype=torch.float32)
        keep = keep.expand(x.numel() // L, L).reshape(x.shape)
        xd = p["x"].dtype
        noised = p["init"].to(xd) + p["renoise"].to(xd) * torch.tensor(p["blend_sigma"], dtype=xd)
        x = torch.where(keep, f(noised), x)
        p["x"].copy_(x.to(p["x"].dtype))
    d = (x - den) * p["inv_sigma"]
    o = p["a"] * x + p["b"] * den + p["g"] * d
    for c, buf in zip(p["c"], p["buf"]):
        if buf is not None:
            o = o + c * f(buf)
    if p["noise"] is not None:
        o = o + p["s"] * f(p["noise"])
    out = {"den": den, "d": d, "x_next": o, "x_in_next": o * p["c_in_next"]}
    for k, v in out.items():
        if p[k] is not None:
            p[k].copy_(v.to(p[k].dtype))
    return out
