"""Pool inputs with many exact ties, shared by the fp32 and the tensor-core pool certification tests."""
import torch


def tie_windows(gen, B, H, W, C):
    """Post-ReLU-like values with many exact ties: each 2x2 window holds 2, 3 or 4 equal positive maxima, or is all zero
    (with -0 mixed in), or is random; values are multiples of 0.25 so equal ones are common anyway."""
    x = torch.randint(0, 8, (B, H, W, C), device="cuda", generator=gen).float() * 0.25
    win = x.reshape(B, H // 2, 2, W // 2, 2, C).permute(0, 1, 3, 5, 2, 4).reshape(B, H // 2, W // 2, C, 4)
    kind = torch.randint(0, 5, win.shape[:4], device="cuda", generator=gen)
    top = win.max(dim=4).values + 0.25
    for k in (2, 3, 4):                                    # k equal maxima at random positions of the window
        sel = kind == k - 2
        order = torch.rand(win.shape, device="cuda", generator=gen).argsort(dim=4)
        hit = order < k
        win = torch.where(sel[..., None] & hit, top[..., None], win)
    zero = kind == 3
    signs = torch.where(torch.rand(win.shape, device="cuda", generator=gen) < 0.5, -0.0, 0.0)
    win = torch.where(zero[..., None], signs, win)
    return win.reshape(B, H // 2, W // 2, C, 2, 2).permute(0, 1, 4, 2, 5, 3).reshape(B, H, W, C).contiguous()
