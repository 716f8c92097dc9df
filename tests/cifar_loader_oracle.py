"""Oracle for the CIFAR loader (test infrastructure only): CifarLoader.__iter__ / AirbenchLoaders of the reference
(utils/dataset.py:101-256) restated in torch, on either device.

The random draws come from torch's default generator in the reference's order; the pixels are moved by plain index
arithmetic (reflect padding and crop windows as gathers) instead of the product's fused kernel.  Pinned on CPU against
``tests/golden/cifar_loader_small.npz`` (written by ``tests/golden/make_cifar_loader_golden.py`` from the reference
itself); the GPU tests and ``tools/cifar_epoch_bench.py`` run it on the device beside the product loader.
"""
import torch

CIFAR_MEAN_STD = {"CIFAR10": ((0.4914, 0.4822, 0.4465), (0.2470, 0.2435, 0.2616)),
                  "CIFAR100": ((0.5071, 0.4867, 0.4408), (0.2675, 0.2565, 0.2761))}


def _reflect_index(n, pad, device):
    """Source index of every position of an n-long axis reflect-padded by pad (edge not repeated): -k -> k, n-1+k -> n-1-k."""
    i = torch.arange(-pad, n + pad, device=device).abs()
    return torch.where(i > n - 1, 2 * (n - 1) - i, i)


def cifar_loader_epochs(images, labels, dataset, batch_size, train, epochs):
    """Yield, per epoch, the list of ``(x, y)`` batches the reference loader makes.

    images uint8 [N, H, W, 3] and labels int64 [N] on the device the draws are made on.  ``train``: AirbenchLoaders'
    training loader (translate 2, random pre-flip on the first epoch, altflip, shuffled, drop_last); otherwise the
    test loader (normalised images in order, last batch partial).  Draw order per epoch: [pre-flip rand(N), first epoch
    only], crop shifts randint(-2, 3, (N, 2)), randperm(N).
    """
    dev = images.device
    mean, std = CIFAR_MEAN_STD[dataset.upper()]
    m = torch.tensor(mean, dtype=torch.float32).view(3, 1, 1).to(dev)
    s = torch.tensor(std, dtype=torch.float32).view(3, 1, 1).to(dev)
    x = images.permute(0, 3, 1, 2) / 255
    x = (x - m) / s
    n, _, h, w = x.shape
    nb = n // batch_size if train else -(-n // batch_size)
    if not train:
        for _ in range(epochs):
            yield [(x[i * batch_size:(i + 1) * batch_size], labels[i * batch_size:(i + 1) * batch_size]) for i in range(nb)]
        return
    r = 2
    pre = torch.rand(n, device=dev) < 0.5
    x = torch.where(pre.view(-1, 1, 1, 1), x.flip(-1), x)
    padded = x[:, :, _reflect_index(h, r, dev)][:, :, :, _reflect_index(w, r, dev)]
    img = torch.arange(n, device=dev).view(n, 1, 1, 1)
    ch = torch.arange(3, device=dev).view(1, 3, 1, 1)
    for e in range(epochs):
        sh = torch.randint(-r, r + 1, size=(n, 2), device=dev)
        rows = (r + sh[:, 0]).view(n, 1, 1, 1) + torch.arange(h, device=dev).view(1, 1, h, 1)
        cols = (r + sh[:, 1]).view(n, 1, 1, 1) + torch.arange(w, device=dev).view(1, 1, 1, w)
        crop = padded[img, ch, rows, cols]
        if e % 2 == 1:
            crop = crop.flip(-1)
        perm = torch.randperm(n, device=dev)
        yield [(crop[perm[i * batch_size:(i + 1) * batch_size]], labels[perm[i * batch_size:(i + 1) * batch_size]])
               for i in range(nb)]
