"""Seeded synthetic frame pairs shaped like the readers' output (data/davis2016_data_utils.py: 384x640 RGB in
[-0.5,0.5], second frame = first frame displaced by a smooth field + noise, GT mask = random blob).  Used by the
benchmark / smoke / tests; no dataset is available offline.  Host side (CPU tensors in pinned memory)."""
import torch
import torch.nn.functional as F


class SyntheticReader(object):
    def __init__(self, height=384, width=640, seed=8964, num_val=16):
        self.h, self.w = height, width
        self.gen = torch.Generator().manual_seed(seed)
        self.val_samples = num_val

    def state(self):
        """The position of the next batch: the generator's state.  restore(state()) makes the following batches repeat."""
        return self.gen.get_state()

    def restore(self, state):
        self.gen.set_state(state)

    def _smooth(self, n, c, amp, div=32):
        lo = torch.randn(n, c, max(self.h // div, 2), max(self.w // div, 2), generator=self.gen)
        return F.interpolate(lo, size=(self.h, self.w), mode='bicubic', align_corners=False) * amp

    def batch(self, n, pinned=True):
        tex = (self._smooth(n, 3, 0.2, 8) + self._smooth(n, 3, 0.15, 64)).clamp(-0.5, 0.5)
        disp = self._smooth(n, 2, 4.0, 64)
        blob = (self._smooth(n, 1, 1.0, 64) > 0.6).float()
        disp = disp * (0.3 + blob)            # the "object" moves more than the background
        ys, xs = torch.meshgrid(torch.linspace(-1, 1, self.h), torch.linspace(-1, 1, self.w), indexing='ij')
        grid = torch.stack([xs, ys], -1).unsqueeze(0) - torch.stack([disp[:, 1] * 2 / self.w, disp[:, 0] * 2 / self.h], -1)
        img2 = F.grid_sample(tex, grid, mode='bilinear', padding_mode='border', align_corners=True)
        img2 = (img2 + 0.01 * torch.randn(img2.shape, generator=self.gen)).clamp(-0.5, 0.5)
        out = [tex.permute(0, 2, 3, 1).contiguous(), img2.permute(0, 2, 3, 1).contiguous(), blob.permute(0, 2, 3, 1).contiguous()]
        if pinned and torch.cuda.is_available():
            out = [t.pin_memory() for t in out]
        names = ['synthetic/seq%02d/%05d.jpg' % (i % 4, i) for i in range(n)]
        return out[0], out[1], out[2], names
