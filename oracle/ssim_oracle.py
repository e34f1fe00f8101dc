"""Functional restatement of the reference's SSIM (modules/commons/ssim.py:319-391) and of the FastSpeech2 task's SSIM
and L1 mel losses (tasks/tts/fs2.py:143-175, tasks/tts/tts.py:124-128).

In float32 on the CPU it is bit-exact to the reference (oracle/gen_golden_ssim.py asserts it).  In float64 it is the
intended function of the same float32 1-D window: the window values are the reference's float32 ones and the 2-D
window is their exact outer product, so it measures what the separable fp32 kernels and eager fp32 conv2d round.
"""
from math import exp

import torch
import torch.nn.functional as F

WINDOW_SIZE = 11
SIGMA = 1.5
C1 = 0.01 ** 2
C2 = 0.03 ** 2


def gaussian(window_size=WINDOW_SIZE, sigma=SIGMA):
    """the reference's float32 1-D window: exp() in double, rounded to float32, over the float32 sum"""
    g = torch.tensor([exp(-(x - window_size // 2) ** 2 / float(2 * sigma ** 2)) for x in range(window_size)],
                     dtype=torch.float32)
    return g / g.sum()


def window(dtype=torch.float32, window_size=WINDOW_SIZE):
    g = gaussian(window_size).to(dtype).unsqueeze(1)
    return g.mm(g.t()).unsqueeze(0).unsqueeze(0)


def ssim_map(img1, img2, window_size=WINDOW_SIZE):
    """[B, 1, H, W] x 2 -> the SSIM map [B, 1, H, W] in the inputs' dtype"""
    w = window(img1.dtype, window_size).to(img1.device)
    p = window_size // 2
    mu1 = F.conv2d(img1, w, padding=p)
    mu2 = F.conv2d(img2, w, padding=p)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = F.conv2d(img1 * img1, w, padding=p) - mu1_sq
    sigma2_sq = F.conv2d(img2 * img2, w, padding=p) - mu2_sq
    sigma12 = F.conv2d(img1 * img2, w, padding=p) - mu1_mu2
    return ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))


def ssim(img1, img2, window_size=WINDOW_SIZE, size_average=True):
    m = ssim_map(img1, img2, window_size)
    return m.mean() if size_average else m.mean(1)


def weights_nonzero_speech(target):
    return target.abs().sum(-1, keepdim=True).ne(0).float().repeat(1, 1, target.size(-1)).to(target.dtype)


def ssim_loss(decoder_output, target, bias=6.0, ssim_fn=ssim):
    """FastSpeech2Task.ssim_loss: decoder_output, target [B, T, n_mel]"""
    weights = weights_nonzero_speech(target)
    l = 1 - ssim_fn(decoder_output[:, None] + bias, target[:, None] + bias, size_average=False)
    return (l * weights).sum() / weights.sum()


def l1_loss(decoder_output, target):
    """FastSpeech2Task.l1_loss"""
    weights = weights_nonzero_speech(target)
    return (F.l1_loss(decoder_output, target, reduction='none') * weights).sum() / weights.sum()


def mel_loss(mel_out, target, loss_and_lambda, ssim_fn=ssim):
    """FastSpeech2Task.add_mel_loss summed over its terms, e.g. {'ssim': 0.5, 'l1': 0.5} in that order"""
    total = 0
    for name, lbd in loss_and_lambda.items():
        l = l1_loss(mel_out, target) if name == 'l1' else ssim_loss(mel_out, target, ssim_fn=ssim_fn)
        total = total + l * lbd
    return total
