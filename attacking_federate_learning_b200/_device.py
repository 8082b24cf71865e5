"""Thin torch-side plumbing: device buffers, current stream, and typed calls into the C ABI.
torch is used for memory and streams only; all arithmetic happens in lib/libafl_b200.so."""
from __future__ import annotations

import torch

from . import _native as nat


def _stream_ptr(t: torch.Tensor):
    return torch.cuda.current_stream(t.device).cuda_stream


def dtype_code(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return nat.AFL_F32
    if t.dtype == torch.bfloat16:
        return nat.AFL_BF16
    if t.dtype == torch.float16:
        return nat.AFL_F16
    raise NotImplementedError(f"users_grads dtype {t.dtype}: only float32, bfloat16 and float16 are supported")


def check_matrix(G: torch.Tensor):
    if not (isinstance(G, torch.Tensor) and G.is_cuda):
        raise TypeError("expected a torch.cuda tensor")
    if G.dim() != 2 or G.stride(1) != 1:
        raise ValueError("users_grads must be a 2-D row-major [clients, params] tensor")
    return G.shape[0], G.shape[1], G.stride(0) if G.shape[0] > 1 else max(G.stride(0), G.shape[1])


class Workspace:
    """Per-device scratch cache (grows on demand, never shrinks)."""
    _cache: dict = {}

    @classmethod
    def get(cls, device, tag: str, nbytes: int) -> torch.Tensor:
        key = (str(device), tag)
        buf = cls._cache.get(key)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=device)
            cls._cache[key] = buf
        return buf


def sqdist_partial(G: torch.Tensor, flags: int = 0, out: torch.Tensor | None = None) -> torch.Tensor:
    """Partial squared-distance table (float64 [n, n]) of this column shard."""
    n, d, ld = check_matrix(G)
    L = nat.lib()
    with torch.cuda.device(G.device):
        nbytes = L.afl_sqdist_workspace_bytes(n, d, dtype_code(G), flags)
        ws = Workspace.get(G.device, "gram", nbytes)
        d2 = out if out is not None else torch.empty((n, n), dtype=torch.float64, device=G.device)
        nat.check(L.afl_sqdist_partial(G.data_ptr(), n, d, ld, dtype_code(G), d2.data_ptr(), ws.data_ptr(), ws.numel(),
                                       flags, _stream_ptr(G)))
    return d2


def sqdist_to_dist(d2: torch.Tensor) -> torch.Tensor:
    n = d2.shape[0]
    dist = torch.empty((n, n), dtype=torch.float32, device=d2.device)
    with torch.cuda.device(d2.device):
        nat.check(nat.lib().afl_sqdist_to_dist(d2.data_ptr(), n, dist.data_ptr(), _stream_ptr(d2)))
    return dist


def krum_select(dist: torch.Tensor, users_count: int, corrupted_count: int, want_scores=False):
    n = dist.shape[0]
    L = nat.lib()
    with torch.cuda.device(dist.device):
        ws = Workspace.get(dist.device, "select", L.afl_select_workspace_bytes(n))
        idx = torch.empty(1, dtype=torch.int32, device=dist.device)
        scores = torch.empty(n, dtype=torch.float32, device=dist.device) if want_scores else None
        nat.check(L.afl_krum_select(dist.data_ptr(), n, users_count, corrupted_count, idx.data_ptr(),
                                    scores.data_ptr() if want_scores else None, ws.data_ptr(), ws.numel(),
                                    _stream_ptr(dist)))
    return (idx, scores) if want_scores else idx


def krum_from_sqdist(d2: torch.Tensor, users_count: int, corrupted_count: int, idx: torch.Tensor | None = None):
    """(all-reduced) squared-distance table -> device int32[1] Krum index, one FFI call."""
    n = d2.shape[0]
    L = nat.lib()
    with torch.cuda.device(d2.device):
        ws = Workspace.get(d2.device, "select", L.afl_select_workspace_bytes(n))
        if idx is None:
            idx = torch.empty(1, dtype=torch.int32, device=d2.device)
        nat.check(L.afl_krum_from_sqdist(d2.data_ptr(), n, users_count, corrupted_count, idx.data_ptr(),
                                         ws.data_ptr(), ws.numel(), _stream_ptr(d2)))
    return idx


def bulyan_select(dist: torch.Tensor, users_count: int, corrupted_count: int) -> torch.Tensor:
    n = dist.shape[0]
    L = nat.lib()
    theta = users_count - 2 * corrupted_count
    with torch.cuda.device(dist.device):
        ws = Workspace.get(dist.device, "select", L.afl_select_workspace_bytes(n))
        sel = torch.empty(max(theta, 1), dtype=torch.int32, device=dist.device)
        nat.check(L.afl_bulyan_select(dist.data_ptr(), n, users_count, corrupted_count, sel.data_ptr(), ws.data_ptr(),
                                      ws.numel(), _stream_ptr(dist)))
    return sel[:max(theta, 0)]


def trimmed_mean(G: torch.Tensor, corrupted_count: int, row_index: torch.Tensor | None = None) -> torch.Tensor:
    n, d, ld = check_matrix(G)
    n_rows = n if row_index is None else int(row_index.numel())
    out = torch.empty(d, dtype=torch.float32, device=G.device)
    with torch.cuda.device(G.device):
        nat.check(nat.lib().afl_trimmed_mean(G.data_ptr(), n, d, ld, dtype_code(G),
                                             None if row_index is None else row_index.data_ptr(), n_rows,
                                             corrupted_count, out.data_ptr(), _stream_ptr(G)))
    return out


def mean(G: torch.Tensor) -> torch.Tensor:
    n, d, ld = check_matrix(G)
    out = torch.empty(d, dtype=torch.float32, device=G.device)
    with torch.cuda.device(G.device):
        nat.check(nat.lib().afl_mean(G.data_ptr(), n, d, ld, dtype_code(G), out.data_ptr(), _stream_ptr(G)))
    return out


def gather_row(G: torch.Tensor, idx_dev: torch.Tensor) -> torch.Tensor:
    n, d, ld = check_matrix(G)
    out = torch.empty(d, dtype=torch.float32, device=G.device)
    with torch.cuda.device(G.device):
        nat.check(nat.lib().afl_gather_row(G.data_ptr(), n, d, ld, dtype_code(G), idx_dev.data_ptr(), out.data_ptr(),
                                           _stream_ptr(G)))
    return out


def alie(G_mal: torch.Tensor, z: float, bcast: torch.Tensor | None = None, alias_mean: bool = True):
    """Returns (crafted, mu, sigma); with alias_mean the returned mu IS crafted (reference aliasing)."""
    f, d, ld = check_matrix(G_mal)
    dev = G_mal.device
    sigma = torch.empty(d, dtype=torch.float32, device=dev)
    crafted = torch.empty(d, dtype=torch.float32, device=dev)
    mu = crafted if alias_mean else torch.empty(d, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        nat.check(nat.lib().afl_alie(G_mal.data_ptr(), f, d, ld, dtype_code(G_mal), float(z), mu.data_ptr(),
                                     sigma.data_ptr(), crafted.data_ptr(),
                                     None if bcast is None else bcast.data_ptr(),
                                     0 if bcast is None else bcast.stride(0), _stream_ptr(G_mal)))
    return crafted, mu, sigma


def alie_band(mu: torch.Tensor, sigma: torch.Tensor, z: float, x: torch.Tensor | None = None,
              out: torch.Tensor | None = None):
    """x is None: mu - z*sigma (malicious.py:35); else np.clip(x, mu - z*sigma, mu + z*sigma) (backdoor.py:60-61)."""
    d = mu.numel()
    for t in (mu, sigma) + (() if x is None else (x,)):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == d):
            raise ValueError("alie_band: contiguous float32 CUDA vectors of equal length expected")
    if out is None:
        out = torch.empty(d, dtype=torch.float32, device=mu.device)
    with torch.cuda.device(mu.device):
        nat.check(nat.lib().afl_alie_band(mu.data_ptr(), sigma.data_ptr(), float(z),
                                          None if x is None else x.data_ptr(), out.data_ptr(), d, _stream_ptr(mu)))
    return out


def momentum_step(weights: torch.Tensor, velocity: torch.Tensor, grads: torch.Tensor, momentum: float, lr: float):
    d = weights.numel()
    with torch.cuda.device(weights.device):
        nat.check(nat.lib().afl_momentum_step(weights.data_ptr(), velocity.data_ptr(), grads.data_ptr(), d,
                                              float(momentum), float(lr), _stream_ptr(weights)))


# ---------------------------------------------------------------------------------------------------------
# multi-GPU exchange over NVLink peer memory (csrc/xgpu.cu)
# ---------------------------------------------------------------------------------------------------------
import ctypes as _C


class PeerContext:
    """One rank's side of the peer-memory exchange: owns the native context and the mapped result words."""

    def __init__(self, world: int, rank: int, n_max: int, device):
        self.world, self.rank, self.n_max, self.device = world, rank, n_max, device
        self.ctx = _C.c_void_p()
        with torch.cuda.device(device):
            nat.check(nat.lib().afl_xgpu_create(world, rank, n_max, _C.byref(self.ctx)))
        self._idx = _C.POINTER(_C.c_int)()
        self._status = _C.POINTER(_C.c_int)()
        self._idx_dev = _C.POINTER(_C.c_int)()

    def handle(self) -> bytes:
        buf = _C.create_string_buffer(64)
        nat.check(nat.lib().afl_xgpu_handle(self.ctx, buf))
        return buf.raw

    def connect(self, handles):
        with torch.cuda.device(self.device):
            nat.check(nat.lib().afl_xgpu_connect(self.ctx, b"".join(handles)))

    def close(self):
        if self.ctx:
            nat.lib().afl_xgpu_destroy(self.ctx)
            self.ctx = _C.c_void_p()

    def krum(self, G: torch.Tensor, users_count: int, corrupted_count: int, flags: int = 0) -> int:
        """Enqueue gram -> publish -> fused tail, synchronise the stream once, return the index.
        (The per-shape plumbing - workspace, dtype code, bound C function - is cached: this is the per-step hot path.)"""
        key = (G.data_ptr(), G.shape, G.stride(0), G.dtype, flags)
        plan = self._plan if getattr(self, "_plan_key", None) == key else None
        if plan is None:
            n, d, ld = check_matrix(G)
            L = nat.lib()
            with torch.cuda.device(G.device):
                ws = Workspace.get(G.device, "gram", L.afl_sqdist_workspace_bytes(n, d, dtype_code(G), flags))
            plan = (L.afl_krum_sharded, n, d, ld, dtype_code(G), ws, _C.byref(self._idx), _C.byref(self._status),
                    _C.byref(self._idx_dev))
            self._plan, self._plan_key = plan, key
        fn, n, d, ld, dt, ws, pidx, pst, pdev = plan
        same_dev = torch.cuda.current_device() == G.device.index
        if not same_dev:
            prev = torch.cuda.current_device()
            torch.cuda.set_device(G.device)
        try:
            stream = torch.cuda.current_stream(G.device)
            rc = fn(self.ctx, G.data_ptr(), n, d, ld, dt, users_count, corrupted_count, ws.data_ptr(), ws.numel(), flags,
                    stream.cuda_stream, pidx, pst, pdev)
            if rc:
                nat.check(rc)
            stream.synchronize()
        finally:
            if not same_dev:
                torch.cuda.set_device(prev)
        if self._status[0] != 0:
            raise RuntimeError("afl_krum_sharded: a peer rank did not publish its partial table in time")
        return int(self._idx[0])

    def allreduce_table(self, G: torch.Tensor, out: torch.Tensor, flags: int = 0) -> torch.Tensor:
        """Partial table of this shard summed over all ranks into `out` ([n, n] float64); enqueues only."""
        n, d, ld = check_matrix(G)
        L = nat.lib()
        with torch.cuda.device(G.device):
            ws = Workspace.get(G.device, "gram", L.afl_sqdist_workspace_bytes(n, d, dtype_code(G), flags))
            nat.check(L.afl_sqdist_allreduce(self.ctx, G.data_ptr(), n, d, ld, dtype_code(G), out.data_ptr(), ws.data_ptr(),
                                             ws.numel(), flags, _stream_ptr(G), _C.byref(self._status)))
        return out
