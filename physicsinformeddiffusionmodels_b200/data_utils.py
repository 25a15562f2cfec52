"""Dataset classes with the reference's names and file formats (reference src/data_utils.py:31-119) and the host -> HBM
staging the training loop needs on the GPU (`DevicePrefetcher`).

* `Dataset`        one CSV per channel, one flattened P*P sample per row -> [N, C, P, P] held in RAM (Darcy study)
* `Dataset_Paths`  one .npy per sample ([65, 65, 10], channels last on disk) -> [10, 65, 65] (mechanics study)
* `DevicePrefetcher` wraps any iterator of CPU batches: the next batch is copied through a pinned staging buffer on a copy
  stream while the current step runs, so the step never waits for PCIe (the reference does `next(dl).to(device)`, a
  synchronous pageable copy, inside the loop: main.py:159)."""
from pathlib import Path

import numpy as np
import pandas as pd
import torch
from torch.utils import data

from .grad_utils import generalized_b_xy_c_to_image, generalized_image_to_b_xy_c  # noqa: F401


def cycle(dl):
    while True:
        for d in dl:
            yield d


class Dataset(data.Dataset):
    def __init__(self, data_directories, use_double=False, return_img=True, gaussian_prior=False):
        super().__init__()
        self.data_paths = list(data_directories)
        dtype = torch.float64 if use_double else torch.float32
        # reference :45-50: channels are stacked on a trailing axis -> [N, P*P, C]
        chans = [pd.read_csv(p, header=None).to_numpy() for p in self.data_paths]
        arr = chans[0] if len(chans) == 1 else np.stack(chans, axis=-1)
        self.data = torch.tensor(arr, dtype=dtype)
        self.num_datapoints = len(self.data)
        if return_img:
            assert len(self.data.shape) == 3, 'Data must be of shape (num_datapoints, pixels_x*pixels_y, channels)'
            self.data = generalized_b_xy_c_to_image(self.data).contiguous()
        if gaussian_prior:
            self.data = torch.randn_like(self.data)          # "no information at all" ablation (reference :62-64)

    def normalize(self, arr, min_val, max_val):
        return (arr - min_val) / (max_val - min_val)

    def unnorm(self, arr, min_val, max_val):
        return arr * (max_val - min_val) + min_val

    def __len__(self):
        return len(self.data)

    def __getitem__(self, index):
        if index >= self.num_datapoints:
            raise IndexError('index out of range')
        return self.data[index]


class Dataset_Paths(data.Dataset):
    def __init__(self, data_directories, use_double=False, return_img=True, gaussian_prior=False, exts=['npy']):
        super().__init__()
        self.paths = [p for ext in exts for p in Path(f'{data_directories}').glob(f'**/*.{ext}')]
        self.paths = sorted(self.paths, key=lambda x: int(x.name.split('.')[0]))      # numeric file-name order (:93)
        self.num_datapoints = len(self.paths)
        self.dtype = torch.float64 if use_double else torch.float32
        self.return_img = return_img
        self.gaussian_prior = gaussian_prior

    def normalize(self, arr, min_val, max_val):
        return (arr - min_val) / (max_val - min_val)

    def unnorm(self, arr, min_val, max_val):
        return arr * (max_val - min_val) + min_val

    def __len__(self):
        return len(self.paths)

    def __getitem__(self, index):
        if index >= self.num_datapoints:
            raise IndexError('index out of range')
        data_np = np.load(self.paths[index], allow_pickle=True, encoding='latin1')
        # on disk: [pixels, pixels, 10] = (vf, strain energy density, von Mises, disp_x, disp_y, E, BC_x, BC_y, load_x, load_y)
        return torch.tensor(data_np.transpose(2, 0, 1), dtype=self.dtype)


class DevicePrefetcher:
    """Iterator adaptor: yields device tensors; batch k+1 travels host -> pinned staging -> HBM on a copy stream while
    the consumer works on batch k.  Two staging / device buffers are recycled (shapes are fixed per loader)."""

    def __init__(self, iterator, device, depth=2):
        self.it = iter(iterator)
        self.device = torch.device(device)
        self.copy_stream = torch.cuda.Stream(device=self.device)
        self.depth = depth
        self._pinned, self._dev, self._events = [None] * depth, [None] * depth, [None] * depth
        self._slot = 0
        self._ready = None
        self._prefetch()

    def _prefetch(self):
        try:
            batch = next(self.it)
        except StopIteration:
            self._ready = None
            return
        k = self._slot
        self._slot = (k + 1) % self.depth
        if self._pinned[k] is None or self._pinned[k].shape != batch.shape or self._pinned[k].dtype != batch.dtype:
            self._pinned[k] = torch.empty(batch.shape, dtype=batch.dtype).pin_memory()
            self._dev[k] = torch.empty(batch.shape, dtype=batch.dtype, device=self.device)
        if self._events[k] is not None:
            self._events[k].synchronize()                    # the staging buffer's previous copy has left the host
        self._pinned[k].copy_(batch)
        with torch.cuda.stream(self.copy_stream):
            # the consumer of this device buffer's previous contents ran on the current stream: order the overwrite
            self.copy_stream.wait_stream(torch.cuda.current_stream(self.device))
            self._dev[k].copy_(self._pinned[k], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self._events[k] = ev
        self._ready = (self._dev[k], ev)

    def __iter__(self):
        return self

    def __next__(self):
        if self._ready is None:
            raise StopIteration
        dev, ev = self._ready
        torch.cuda.current_stream(self.device).wait_event(ev)
        self._prefetch()
        return dev
