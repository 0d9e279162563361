"""Image losses of GaussianSplatting3D.training (main_3DGS.py:184-192): L1 + lambda_alpha * MSE(alpha) +
lambda_ssim * (1 - MS-SSIM).  MS-SSIM restates pytorch_msssim.MS_SSIM(data_range=1, size_average=True,
channel=3) (win 11, sigma 1.5, 5 scales, weights .0448/.2856/.3001/.2363/.1333, K=(0.01,0.03)); torch ops only —
the loss sits beside the hot path (SURVEY §8f), its gradient wrt the rendered image feeds the rasterizer backward."""
import torch
import torch.nn.functional as F

_MS_WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)


def _gauss_1d(size=11, sigma=1.5, device=None, dtype=torch.float32):
    c = torch.arange(size, dtype=dtype, device=device) - size // 2
    g = torch.exp(-(c ** 2) / (2 * sigma ** 2))
    return g / g.sum()


def _filter(x, win):
    C = x.shape[1]
    k = win.view(1, 1, -1, 1).repeat(C, 1, 1, 1)
    x = F.conv2d(x, k, groups=C)
    return F.conv2d(x, k.transpose(2, 3), groups=C)


def _ssim_cs(X, Y, win, data_range=1.0, K=(0.01, 0.03)):
    C1, C2 = (K[0] * data_range) ** 2, (K[1] * data_range) ** 2
    mu1, mu2 = _filter(X, win), _filter(Y, win)
    mu1_sq, mu2_sq, mu12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s1 = _filter(X * X, win) - mu1_sq
    s2 = _filter(Y * Y, win) - mu2_sq
    s12 = _filter(X * Y, win) - mu12
    cs_map = (2 * s12 + C2) / (s1 + s2 + C2)
    ssim_map = ((2 * mu12 + C1) / (mu1_sq + mu2_sq + C1)) * cs_map
    return ssim_map.flatten(2).mean(-1), cs_map.flatten(2).mean(-1)


def ms_ssim(X, Y, data_range=1.0, size_average=True):
    """X, Y: [B,C,H,W]; the smaller side must exceed (11-1)*2^4 = 160 (as the package asserts)."""
    if min(X.shape[-2:]) <= (11 - 1) * 2 ** 4:
        raise ValueError("Image size should be larger than 160 due to the 4 downsamplings in ms-ssim")
    win = _gauss_1d(device=X.device, dtype=X.dtype)
    w = torch.tensor(_MS_WEIGHTS, device=X.device, dtype=X.dtype)
    mcs = []
    for i in range(5):
        ssim_pc, cs = _ssim_cs(X, Y, win, data_range)
        if i < 4:
            mcs.append(torch.relu(cs))
            pad = [s % 2 for s in X.shape[2:]]
            X = F.avg_pool2d(X, kernel_size=2, padding=pad)
            Y = F.avg_pool2d(Y, kernel_size=2, padding=pad)
    vals = torch.stack(mcs + [torch.relu(ssim_pc)], dim=0)                   # [5,B,C]
    out = torch.prod(vals ** w.view(-1, 1, 1), dim=0)
    return out.mean() if size_average else out.mean(1)


def training_loss(images, alphas, ref_images, ref_masks, lambda_ssim=0.2, lambda_alpha=3.0):
    """images [B,3,H,W], alphas [B,1,H,W], ref_images [B,3,H,W], ref_masks [B,1,H,W] -> scalar (main_3DGS.py:184-192)."""
    img_m = images * ref_masks
    ref_m = ref_images * ref_masks
    loss = (1 - lambda_ssim) * F.l1_loss(img_m, ref_m) + lambda_alpha * F.mse_loss(alphas, ref_masks)
    if lambda_ssim > 0:
        loss = loss + lambda_ssim * (1 - ms_ssim(ref_m, img_m))
    return loss
