"""float64 reference of ``tl_lora_apply`` (``include/tiny_llm_b200.h``) that keeps the contract's rounding points, the
error bound the kernel is held to, and the CPU stand-in of ``ext.lora_apply`` for the host tests.

Per row with adapter ``a >= 0`` and targeted segment ``s``:
    t_j = bf16(sum_i A[j,i] x_i)        d_o = sc * sum_j B[o,j] t_j        y_o = bf16(base_o + d_o)      x'_o = bf16(res_o + y_o)
The kernel runs the two sums in fp32.  Its error against the float64 value has no absolute term:
  * each t_j is off by at most e_j = N u sum_i |A[j,i] x_i| (u = 2^-24) before rounding; where the float64 sum lies within
    e_j of a bf16 rounding boundary the rounded t_j may land one bf16 step away, which moves d_o by sc |B[o,j]| step(t_j);
  * the expand sum adds (r + 1) u sc sum_j |B[o,j] t_j|;
  * y and x' are each rounded once more: one bf16 step of the reference value where d's error can cross a boundary.
"""

import torch

U = 2.0**-24


def bf16_round(v: torch.Tensor) -> torch.Tensor:
    """float64 -> nearest bf16 (ties to even) -> float64."""
    return v.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def bf16_step(v: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at |v| (8 significant bits), never below the smallest normal's."""
    mag = v.abs().clamp_min(2.0**-126)
    return torch.exp2(torch.floor(torch.log2(mag)) - 7)


def _near_boundary(v: torch.Tensor, err: torch.Tensor) -> torch.Tensor:
    """Whether v lies within err of a midpoint between two neighbouring bf16 values."""
    step = bf16_step(v)
    frac = torch.remainder(v / step, 1.0)
    return (frac - 0.5).abs() * step <= err


def lora_reference(x, ys, ids, site, residual=None):
    """Reference outputs and per-element bounds.  ``x`` bf16 [M, N]; ``ys`` one bf16 [M, K_s] per segment (the base
    projection); ``site`` an ``ext.LoraSite`` on the CPU.  Returns ``(outs, bounds)``, float64 lists per segment; rows
    with a negative id and untargeted segments get bound 0 (their bits are the base's, or the one residual add)."""
    M = x.shape[0]
    x64 = x.to(torch.float64)
    rs = None if residual is None else [r.to(torch.float64) for r in residual]
    outs = [y.to(torch.float64).clone() for y in ys]
    bounds = [torch.zeros_like(o) for o in outs]
    rmax = site.r_max
    for m in range(M):
        a = int(ids[m])
        if a >= 0:
            r, sc, mask = int(site.ranks[a]), float(site.scales[a]), int(site.seg_mask[a])
            for s in range(site.nseg):
                if not (mask >> s) & 1:
                    continue
                A = site.a[a, s * rmax : s * rmax + r].to(torch.float64)
                B = site.b[s][a, :, :r].to(torch.float64)
                t_exact = A @ x64[m]
                e_t = site.N * U * (A.abs() @ x64[m].abs())
                t = bf16_round(t_exact)
                flip = torch.where(_near_boundary(t_exact, e_t), bf16_step(t_exact), torch.zeros_like(t))
                d = sc * (B @ t)
                e_d = abs(sc) * (B.abs() @ flip + (r + 1) * U * (B.abs() @ t.abs()))
                y_exact = outs[s][m] + d
                y = bf16_round(y_exact)
                outs[s][m] = y
                bounds[s][m] = e_d + torch.where(_near_boundary(y_exact, e_d), bf16_step(y_exact), torch.zeros_like(y))
        if rs is not None:
            for s in range(site.nseg):
                z_exact = rs[s][m] + outs[s][m]
                e = bounds[s][m]
                outs[s][m] = bf16_round(z_exact)
                bounds[s][m] = e + torch.where(_near_boundary(z_exact, e) & (e > 0), bf16_step(z_exact), torch.zeros_like(e))
    return outs, bounds


def lora_apply_like_ext(x, y, adapter_ids, site, residual=None, stream=None):
    """CPU stand-in of ``ext.lora_apply``: the reference's values written into ``y`` in place."""
    from extensions_b200 import tiny_llm_ext_b200 as ext

    M, ys, rs = ext._lora_args(x, y, adapter_ids, site, residual)
    outs, _ = lora_reference(x.reshape(M, -1), ys, adapter_ids.tolist(), site, rs)
    for dst, src in zip(ys, outs):
        dst.copy_(src.to(torch.bfloat16))
    return y


def install(ext_module, monkeypatch) -> None:
    monkeypatch.setattr(ext_module, "lora_apply", lora_apply_like_ext)


def random_site(gen, N, Ks, ranks, r_max=None, masks=None, device="cpu"):
    """A site of ``len(ranks)`` random adapters (A ~ N(0, 1/N), B ~ N(0, 0.05^2), scale 2), each padded to ``r_max``."""
    from extensions_b200 import tiny_llm_ext_b200 as ext

    n, nseg = len(ranks), len(Ks)
    r_max = r_max or max(ranks)
    A = torch.zeros((n, nseg * r_max, N), dtype=torch.bfloat16)
    Bs = [torch.zeros((n, K, r_max), dtype=torch.bfloat16) for K in Ks]
    for i, r in enumerate(ranks):
        for s in range(nseg):
            A[i, s * r_max : s * r_max + r] = (torch.randn(r, N, generator=gen) * N**-0.5).to(torch.bfloat16)
            Bs[s][i, :, :r] = (torch.randn(Ks[s], r, generator=gen) * 0.05).to(torch.bfloat16)
    masks = masks if masks is not None else [(1 << nseg) - 1] * n
    return ext.LoraSite(A.to(device), [b.to(device) for b in Bs], torch.full((n,), 2.0, dtype=torch.float32, device=device),
                        torch.tensor(ranks, dtype=torch.int32, device=device), torch.tensor(masks, dtype=torch.int32, device=device))


def site_to(site, device):
    from extensions_b200 import tiny_llm_ext_b200 as ext

    return ext.LoraSite(site.a.to(device), [b.to(device) for b in site.b], site.scales.to(device), site.ranks.to(device), site.seg_mask.to(device))
