"""torchmetrics 1.3.2 `_compute_fid`, restated from memory [3P-mem]: not pinned against the package, which is not
installed here."""
import torch


def _compute_fid(mu1, sigma1, mu2, sigma2):
    a = (mu1 - mu2).square().sum(dim=-1)
    b = sigma1.trace() + sigma2.trace()
    c = torch.linalg.eigvals(sigma1 @ sigma2).sqrt().real.sum(dim=-1)
    return a + b - 2 * c
