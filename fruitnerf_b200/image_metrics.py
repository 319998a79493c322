"""Full-image evaluation metrics and visualisation images of ``FruitModel.get_image_metrics_and_images``
(fruit_nerf/fruit_nerf.py:403-458).  Evaluation-time host code over one rendered [H,W,*] image -- outside the per-ray
hot path, so plain torch on whatever device the outputs live on (``get_outputs_for_camera_ray_bundle`` returns CPU
tensors, as upstream).

The reference takes these from third-party packages that are absent offline; what is restated here:

* ``psnr``  -- torchmetrics ``PeakSignalNoiseRatio(data_range=1.0)``: 10 log10(1 / mse).
* ``ssim``  -- torchmetrics ``structural_similarity_index_measure`` with its defaults (11x11 gaussian window, sigma 1.5,
  k1 0.01, k2 0.03, data_range = the larger value range of the two inputs, reflect padding, border cropped, mean).
* ``binary_jaccard`` -- torchmetrics ``BinaryJaccardIndex()`` (threshold 0.5 on float predictions).
* ``apply_colormap`` / ``apply_depth_colormap`` -- nerfstudio ``utils.colormaps`` (turbo for one-channel images; depth
  normalised to its own min / max and faded to white by 1 - accumulation).  nerfstudio indexes matplotlib's 256-entry
  turbo table; matplotlib is absent here, so the table is rebuilt from the published degree-5 polynomial fit of turbo (close to
  the table in the interior, visibly off at the two ends): these are pictures for a viewer / logger, not parity outputs.
  The `render` command's frame kernel (fnr_compose_frame) is handed this same table.
* ``restated_image_scores`` -- the record the `eval` command's device kernels (fnr_image_stats, fnr_ssim) write for one
  view, in fp64: the tests' reference for them.
* LPIPS needs the pretrained AlexNet weights torchmetrics downloads: not restated; the key is omitted.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor


def psnr(preds: Tensor, target: Tensor, data_range: float = 1.0) -> Tensor:
    mse = torch.mean((preds.float() - target.float()) ** 2)
    return 10.0 * torch.log10(data_range ** 2 / mse)


def _gaussian_window(kernel_size: int, sigma: float, dtype, device) -> Tensor:
    dist = torch.arange((1 - kernel_size) / 2, (1 + kernel_size) / 2, 1, dtype=dtype, device=device)
    g = torch.exp(-((dist / sigma) ** 2) / 2)
    return (g / g.sum())[None, :]  # [1, k]


def ssim(preds: Tensor, target: Tensor, kernel_size: int = 11, sigma: float = 1.5, data_range: Optional[float] = None, k1: float = 0.01,
         k2: float = 0.03) -> Tensor:
    """preds / target [B,C,H,W] -> mean SSIM over the batch."""
    if preds.shape != target.shape or preds.dim() != 4:
        raise ValueError(f"expected two [B,C,H,W] tensors of the same shape, got {tuple(preds.shape)} and {tuple(target.shape)}")
    preds, target = preds.float(), target.float()
    if data_range is None:
        data_range = float(max(preds.max() - preds.min(), target.max() - target.min()))
    c1, c2 = (k1 * data_range) ** 2, (k2 * data_range) ** 2
    C = preds.shape[1]
    pad = (kernel_size - 1) // 2
    g = _gaussian_window(kernel_size, sigma, preds.dtype, preds.device)
    kernel = (g.t() @ g).expand(C, 1, kernel_size, kernel_size)
    p = F.pad(preds, (pad, pad, pad, pad), mode="reflect")
    t = F.pad(target, (pad, pad, pad, pad), mode="reflect")
    stack = torch.cat((p, t, p * p, t * t, p * t))  # [5B, C, H+2p, W+2p]
    out = F.conv2d(stack, kernel, groups=C)
    mu_p, mu_t, pp, tt, pt = out.split(preds.shape[0])
    mu_pp, mu_tt, mu_pt = mu_p * mu_p, mu_t * mu_t, mu_p * mu_t
    sig_p, sig_t, sig_pt = pp - mu_pp, tt - mu_tt, pt - mu_pt
    upper, lower = 2 * sig_pt + c2, sig_p + sig_t + c2
    full = ((2 * mu_pt + c1) * upper) / ((mu_pp + mu_tt + c1) * lower)
    full = full[..., pad:-pad, pad:-pad] if pad else full
    return full.reshape(full.shape[0], -1).mean(-1).mean()


def binary_jaccard(preds: Tensor, target: Tensor, threshold: float = 0.5) -> Tensor:
    """|pred AND target| / |pred OR target| with float predictions thresholded at ``threshold`` (0 when both are empty)."""
    p = preds > threshold if preds.is_floating_point() else preds.bool()
    t = target > 0.5 if target.is_floating_point() else target.bool()
    inter = (p & t).sum().float()
    union = (p | t).sum().float()
    return torch.where(union > 0, inter / union.clamp_min(1), torch.zeros_like(union))


def _turbo_table(device) -> Tensor:
    x = torch.linspace(0.0, 1.0, 256, dtype=torch.float64)
    v4 = torch.stack([torch.ones_like(x), x, x * x, x ** 3], dim=-1)
    v2 = torch.stack([x ** 4, x ** 5], dim=-1)
    r4, g4, b4 = (0.13572138, 4.61539260, -42.66032258, 132.13108234), (0.09140261, 2.19418839, 4.84296658, -14.18503333), \
        (0.10667330, 12.64194608, -60.58204836, 110.36276771)
    r2, g2, b2 = (-152.94239396, 59.28637943), (4.27729857, 2.82956604), (-89.90310912, 27.34824973)
    rgb = torch.stack([v4 @ torch.tensor(c4, dtype=torch.float64) + v2 @ torch.tensor(c2, dtype=torch.float64)
                       for c4, c2 in ((r4, r2), (g4, g2), (b4, b2))], dim=-1)
    return rgb.clamp(0, 1).float().to(device)


def apply_colormap(image: Tensor) -> Tensor:
    """nerfstudio colormaps.apply_colormap with default options: [..,3] passes through, [..,1] float -> turbo."""
    if image.shape[-1] == 3:
        return image
    if image.shape[-1] != 1 or not image.is_floating_point():
        raise NotImplementedError(f"colormap of a {tuple(image.shape)} {image.dtype} image")
    idx = (torch.nan_to_num(image, 0).clamp(0, 1) * 255).long()[..., 0]
    return _turbo_table(image.device)[idx]


def apply_depth_colormap(depth: Tensor, accumulation: Optional[Tensor] = None, near_plane: Optional[float] = None,
                         far_plane: Optional[float] = None) -> Tensor:
    """``near_plane or min(depth)``, ``far_plane or max(depth)`` as nerfstudio writes it: a plane of 0 also means the
    depth's own extreme."""
    near, far = near_plane or float(torch.min(depth)), far_plane or float(torch.max(depth))
    d = torch.clip((depth - near) / (far - near + 1e-10), 0, 1)
    colored = apply_colormap(d)
    if accumulation is not None:
        colored = colored * accumulation + (1 - accumulation)
    return colored


def image_metrics_and_images(outputs: Dict[str, Tensor], batch: Dict[str, Tensor], num_proposal_iterations: int, device) -> Tuple[Dict, Dict]:
    """Body of FruitModel.get_image_metrics_and_images (fruit_nerf.py:403-458), key for key."""
    image = batch["image"].to(device)
    rgb = torch.clamp(outputs["rgb"].to(device), min=0, max=1)
    accumulation = outputs["accumulation"].to(device)
    acc = apply_colormap(accumulation)
    depth = apply_depth_colormap(outputs["depth"].to(device), accumulation=accumulation)
    images = {"img": torch.cat([image, rgb], dim=1), "accumulation": acc, "depth": depth}
    im, pr = torch.moveaxis(image, -1, 0)[None, ...], torch.moveaxis(rgb, -1, 0)[None, ...]  # [H,W,C] -> [1,C,H,W]
    metrics = {"psnr": float(psnr(im, pr)), "ssim": float(ssim(im, pr))}
    for i in range(num_proposal_iterations):
        key = f"prop_depth_{i}"
        if key in outputs:
            images[key] = apply_depth_colormap(outputs[key].to(device), accumulation=accumulation)
    sem = outputs["semantics"].to(device)
    images["semantics_colormap"] = torch.sigmoid(sem)  # fruit_nerf.py:440-443
    mask = batch["fruit_mask"].to(device)
    images["fruit_mask"] = mask.repeat(1, 1, 3)
    # fruit_nerf.py:451-455, literally: `F.softmax(outputs["semantics"])` WITHOUT a dim on the [H,W,1] logits.  torch's legacy rule
    # picks dim 0 for 3-d inputs, so the "probability" is a softmax over the image ROWS (values ~1/H, never above 0.5 once H > 2)
    # and the logged `iou` is ~0 whatever the render shows.  Kept under the reference's key for parity; `fruit_iou` is the useful one:
    # |sigmoid(logit) > 0.9 AND mask| / |... OR mask|, the thresholding get_outputs applies (fruit_nerf.py:349-351).
    metrics["iou"] = float(binary_jaccard(torch.softmax(sem, dim=0)[..., 0], mask[..., 0]))
    metrics["fruit_iou"] = float(binary_jaccard((torch.sigmoid(sem) > 0.9)[..., 0], mask[..., 0])) if float(mask.sum()) or bool(
        (torch.sigmoid(sem) > 0.9).any()) else 1.0
    return metrics, images


def restated_image_scores(rgb: Tensor, semantics: Tensor, accumulation: Tensor, image: Tensor, fruit_mask: Tensor) -> Dict[str, float]:
    """What ``ops.image_stats`` and ``ops.image_ssim`` (fnr_metrics.cu) write into their record, restated in fp64 torch
    on the inputs' device (the tests' reference; keys ``_lib.IMAGE_RECORD_FIELDS``).  ``rgb`` as rendered ([H*W,3] or
    [H,W,3]), ``semantics`` logits, ``accumulation``, ``image`` [H,W,3] and ``fruit_mask`` [H,W,1], all fp32.
    The SSIM is torchmetrics' with NO padding: the window runs over the unpadded images and the (H - 10) x (W - 10) map
    that results is exactly the interior ``ssim`` above keeps after its crop, because a kept pixel's window never
    reaches the reflect-padded border."""
    H, W = image.shape[:2]
    if H < 11 or W < 11:
        raise ValueError(f"a {W}x{H} image is smaller than the 11x11 SSIM window")
    x32 = torch.clamp(rgb.float().reshape(H, W, 3), min=0, max=1)
    y32 = image.float().reshape(H, W, 3)
    x, y = x32.double(), y32.double()
    pred = (torch.sigmoid(semantics.float()) > 0.9).reshape(-1)
    truth = (fruit_mask.float() > 0.5).reshape(-1)
    out = {"sse": float(((x - y) ** 2).sum()), "rgb_min": float(x32.min()), "rgb_max": float(x32.max()), "image_min": float(y32.min()),
           "image_max": float(y32.max()), "accumulation_sum": float(accumulation.double().sum()),
           "fruit_tp": float((pred & truth).sum()), "fruit_fp": float((pred & ~truth).sum()), "fruit_fn": float((~pred & truth).sum()),
           "fruit_tn": float((~pred & ~truth).sum())}
    data_range = float(torch.maximum(x32.max() - x32.min(), y32.max() - y32.min()))  # fp32 differences, as torchmetrics
    c1, c2 = (0.01 * data_range) ** 2, (0.03 * data_range) ** 2
    g = _gaussian_window(11, 1.5, torch.float64, x.device)  # [1, 11]
    xc, yc = x.permute(2, 0, 1)[:, None], y.permute(2, 0, 1)[:, None]  # [3,1,H,W]
    stack = torch.cat((xc, yc, xc * xc, yc * yc, xc * yc))
    rows = F.conv2d(stack, g[None, None])  # horizontal 11 taps, then vertical
    mu_x, mu_y, xx, yy, xy = F.conv2d(rows, g.t()[None, None]).split(3)
    mxx, myy, mxy = mu_x * mu_x, mu_y * mu_y, mu_x * mu_y
    full = ((2 * mxy + c1) * (2 * (xy - mxy) + c2)) / ((mxx + myy + c1) * ((xx - mxx) + (yy - myy) + c2))
    out["ssim"] = float(full.sum() / full.numel())
    out["data_range"] = data_range
    return out
