"""normalizer.py: the observation / goal statistics on the device, float32 like the reference's TF variables.
`state` is [sum(size) | sumsq(size) | count] with count starting at 1 (tf.ones_initializer); mean starts at 0 and std
at 1.  The update over newly stored episodes and recompute_stats run as one kernel (ops.her_norm, csrc/her.cu)."""
from collections import OrderedDict

import torch


class Normalizer:
    def __init__(self, size, eps=1e-2, default_clip_range=float('inf'), device=None):
        self.size, self.eps, self.default_clip_range = int(size), eps, default_clip_range
        f32 = dict(dtype=torch.float32, device=device)
        self.state = torch.zeros(2 * self.size + 1, **f32)
        self.state[2 * self.size] = 1.0
        self.mean = torch.zeros(self.size, **f32)
        self.std = torch.ones(self.size, **f32)

    @property
    def tensors(self):
        return self.state, self.mean, self.std

    def tf_variables(self, scope):
        st = self.state.cpu().numpy()
        D = self.size
        return OrderedDict([(f'{scope}/sum:0', st[:D].copy()), (f'{scope}/sumsq:0', st[D:2 * D].copy()),
                            (f'{scope}/count:0', st[2 * D:].copy()), (f'{scope}/mean:0', self.mean.cpu().numpy()),
                            (f'{scope}/std:0', self.std.cpu().numpy())])

    def load_tf(self, values, scope):
        D = self.size
        for name, sl in (('sum', slice(0, D)), ('sumsq', slice(D, 2 * D)), ('count', slice(2 * D, 2 * D + 1))):
            self.state[sl] = torch.as_tensor(values[f'{scope}/{name}:0'], dtype=torch.float32).reshape(-1)
        self.mean.copy_(torch.as_tensor(values[f'{scope}/mean:0'], dtype=torch.float32))
        self.std.copy_(torch.as_tensor(values[f'{scope}/std:0'], dtype=torch.float32))
