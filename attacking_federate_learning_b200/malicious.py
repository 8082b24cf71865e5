"""Drop-in for the reference's `malicious.py` (Attack / DriftAttack, the "A Little Is Enough"
perturbation) and for the gradient-crafting half of `backdoor.py` (BackdoorAttack._attack_grads),
backed by the fused mu/sigma/perturb kernel `afl_alie` and the band kernel `afl_alie_band`.

Reference surface mirrored: Attack.__init__/attack (malicious.py:4-27), DriftAttack._attack_grads
(malicious.py:30-36), BackdoorAttack._attack_grads (backdoor.py:52-63; the network training it calls,
backdoor.py:108-, is model code and out of scope: the caller passes it in).  `users` are duck-typed
objects with `.grads`, `.original_params`, `.learning_rate` exactly as the reference expects; `.grads`
may be NumPy float32 vectors or torch.cuda vectors.  As in the reference, after `attack()` every
malicious user holds THE SAME array object; for DriftAttack that object is also `self.grads_mean`
(mutated in place); `self.grads_stdev` keeps sigma.  All arithmetic runs on the GPU.  With NumPy
gradients `attack()` streams column slabs of the users' own arrays to the device (`afl_alie_host`, within
the host-buffer budget of `defences.py`), so no stacked f x D copy exists on the host or the device; the
statistics come back as NumPy vectors.  `attack_rows` is the GPU-resident form for a stacked matrix whose rows 0..f-1
are the malicious users: the fused drift kernel for DriftAttack, and for BackdoorAttack the backdoor kernels around
one call of the training (`batched.backdoor_rows` with one problem).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as nat


def _is_cuda(x):
    import torch
    return isinstance(x, torch.Tensor) and x.is_cuda


def _host_rows(users):
    """The users' gradients as C-contiguous 1-D float32 arrays; only arrays that are not already so are converted."""
    rows = []
    for u in users:
        g = u.grads
        if not (isinstance(g, np.ndarray) and g.dtype == np.float32 and g.ndim == 1 and g.flags.c_contiguous):
            g = np.ascontiguousarray(np.asarray(g, np.float32))
        if g.ndim != 1:
            raise ValueError("users' grads must be 1-D vectors")
        if rows and g.shape != rows[0].shape:
            raise ValueError("all input arrays must have the same shape")       # what np.stack raises
        rows.append(g)
    return rows


def _host_alie(users, z, crafted: bool):
    """(mu, sigma) of the users' NumPy gradients, one afl_alie_host call.  crafted=True: mu is overwritten in place
    by mu - z*sigma (the reference's aliasing); otherwise z is unused."""
    rows = _host_rows(users)
    f, d = len(rows), rows[0].size
    mu, sigma = np.empty(d, np.float32), np.empty(d, np.float32)
    ptrs = (C.c_void_p * f)(*[r.ctypes.data for r in rows])
    nat.check(nat.lib().afl_alie_host(ptrs, f, d, float(z), mu.ctypes.data, sigma.ctypes.data,
                                      mu.ctypes.data if crafted else None, 0))
    return mu, sigma


def _to_dev(x):
    import torch
    if _is_cuda(x):
        return x.contiguous() if x.dtype == torch.float32 else x.float().contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x, np.float32))).cuda()


class Attack(object):
    def __init__(self, num_std):
        self.num_std = num_std
        self.grads_mean = None
        self.grads_stdev = None

    def attack(self, users):
        if len(users) == 0:
            return
        fused = self.num_std != 0 and self._fused_drift()
        # malicious.py:17-18 (mu, sigma); with the fused DriftAttack also malicious.py:35 in the same pass
        if _is_cuda(users[0].grads):
            import torch
            from . import _device as dev
            rows = torch.stack([u.grads for u in users])
            _, self.grads_mean, self.grads_stdev = dev.alie(rows, self.num_std if fused else 0.0, None, alias_mean=fused)
        else:
            self.grads_mean, self.grads_stdev = _host_alie(users, self.num_std if fused else 0.0, fused)
        if self.num_std == 0:                               # malicious.py:20-21: statistics only
            return
        if fused:
            mal_grads = self.grads_mean                     # the reference returns grads_mean itself
        else:                                               # malicious.py:23: the template-method hook
            mal_grads = self._attack_grads(self.grads_mean, self.grads_stdev, users[0].original_params,
                                           users[0].learning_rate)
        for usr in users:
            usr.grads = mal_grads

    def _fused_drift(self):
        return False

    def _attack_grads(self, grads_mean, grads_stdev, original_params, learning_rate):
        raise NotImplementedError

    def attack_rows(self, users_grads, corrupted_count):
        """GPU-resident form: the malicious users are rows 0..f-1 of the stacked matrix (main.py:28);
        computes the crafted vector and writes it into those rows in place (what server.py:82-83 does
        next with the aliased `usr.grads`).  Returns the crafted vector."""
        from . import _device as dev
        if corrupted_count <= 0:
            return None
        mal = users_grads[:corrupted_count]
        if self.num_std == 0:
            _, mu, sigma = dev.alie(mal, 0.0, None, alias_mean=False)
            self.grads_mean, self.grads_stdev = mu, sigma
            return None
        import torch
        bcast = users_grads if users_grads.dtype == torch.float32 else None
        crafted, mu, sigma = dev.alie(mal, self.num_std, bcast, alias_mean=True)
        if bcast is None:
            users_grads[:corrupted_count] = crafted.to(users_grads.dtype)
        self.grads_mean, self.grads_stdev = mu, sigma
        return crafted


class DriftAttack(Attack):
    def __init__(self, num_std):
        super(DriftAttack, self).__init__(num_std)

    def _fused_drift(self):
        # one pass over the malicious rows does mu, sigma and mu - z*sigma unless a subclass replaced the hook
        return type(self)._attack_grads is DriftAttack._attack_grads

    def _attack_grads(self, grads_mean, grads_stdev, original_params, learning_rate):
        # malicious.py:34-36  `grads_mean[:] -= self.num_std * grads_stdev[:]`, in place, on the device
        from . import _device as dev
        if _is_cuda(grads_mean):
            dev.alie_band(grads_mean, _to_dev(grads_stdev), self.num_std, None, out=grads_mean)
        else:
            grads_mean[:] = dev.alie_band(_to_dev(grads_mean), _to_dev(grads_stdev), self.num_std).cpu().numpy()
        return grads_mean


class BackdoorAttack(Attack):
    """backdoor.py:13-63 without the model: `train_malicious_network(initial_params_flat) -> params`
    (backdoor.py:108) is supplied by the caller (any callable; it receives and returns the type of
    `original_params`)."""

    def __init__(self, num_std, train_malicious_network):
        super(BackdoorAttack, self).__init__(num_std)
        self.train_malicious_network = train_malicious_network

    def _attack_grads(self, grads_mean, grads_stdev, original_params, learning_rate):
        from . import _device as dev
        on_gpu = _is_cuda(grads_mean)
        mu, sd, w = _to_dev(grads_mean), _to_dev(grads_stdev), _to_dev(original_params)
        step = mu * learning_rate                                  # fp32 product, as NumPy's weak scalar
        initial = w - step                                         # backdoor.py:54
        mal = self.train_malicious_network(initial if on_gpu else initial.cpu().numpy())   # backdoor.py:56
        new_params = _to_dev(mal) + step                           # backdoor.py:59
        import torch
        # a 0-d tensor divisor: torch turns division by a Python scalar into a multiplication by 1/lr
        new_grads = (initial - new_params) / torch.tensor(learning_rate, dtype=torch.float32, device=mu.device)   # backdoor.py:60
        out = dev.alie_band(mu, sd, self.num_std, new_grads.contiguous())            # backdoor.py:62-63
        return out if on_gpu else out.cpu().numpy()

    def attack_rows(self, users_grads, corrupted_count, original_params=None, learning_rate=None):
        """GPU-resident form of attack() (backdoor.py:52-63): the malicious users are rows 0..f-1 of the stacked
        matrix (main.py:28); `original_params` (fp32 CUDA [D]) and `learning_rate` are what users[0] carries.  Computes
        the statistics and the crafted vector on the device, calling `train_malicious_network` once in between with
        a fp32 CUDA [D] vector (it must return one), and writes the crafted vector into those rows in place
        (server.py:82-83).  Sets grads_mean and grads_stdev and returns the crafted vector; None when
        corrupted_count <= 0, and None after the statistics when num_std == 0 (malicious.py:20-21)."""
        if corrupted_count <= 0:                            # malicious.py:11-12: no malicious user, nothing to craft
            return None
        if original_params is None or learning_rate is None:
            raise TypeError("BackdoorAttack.attack_rows needs original_params and learning_rate (backdoor.py:52)")
        import torch
        from . import batched

        def train(initial, problems):
            mal = self.train_malicious_network(initial[0])
            return mal[None] if isinstance(mal, torch.Tensor) else mal
        crafted, mu, sigma = batched.backdoor_rows(users_grads[None], corrupted_count, self.num_std, original_params,
                                                   learning_rate, train)
        self.grads_mean, self.grads_stdev = mu[0], sigma[0]
        return None if self.num_std == 0 else crafted[0]


def backdoor_clip(new_grads, grads_mean, grads_stdev, num_std):
    """np.clip(new_grads, grads_mean - num_std*grads_stdev, grads_mean + num_std*grads_stdev) (backdoor.py:62-63)."""
    from . import _device as dev
    out = dev.alie_band(_to_dev(grads_mean), _to_dev(grads_stdev), num_std, _to_dev(new_grads))
    return out if _is_cuda(new_grads) else out.cpu().numpy()
