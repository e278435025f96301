"""Shared test helpers: seeded inputs, oracle-side evaluation of one layer, stored results of the
compiled reference (tests/golden/)."""
import hashlib
import os

import numpy as np
import torch

from oracle import oracle_np as O


def random_cloud(n, extent, seed, D=3, batches=1, allow_negative=False):
    g = torch.Generator().manual_seed(seed)
    lo = -extent if allow_negative else 0
    c = torch.randint(lo, extent, (n, D), generator=g, dtype=torch.int32)
    b = torch.randint(0, batches, (n, 1), generator=g, dtype=torch.int32)
    return torch.cat([b, c], 1)


def unique_cloud(n, extent, seed, D=3, batches=1, allow_negative=False):
    c = random_cloud(n, extent, seed, D, batches, allow_negative)
    return torch.unique(c, dim=0)[torch.randperm(
        len(torch.unique(c, dim=0)), generator=torch.Generator().manual_seed(seed + 1))]


def kmap_lists(kdict, K):
    """{k: IntTensor[2,n]} -> (in_maps, out_maps) numpy lists of length K."""
    im, om = [], []
    for k in range(K):
        if k in kdict:
            t = kdict[k].cpu().numpy().astype(np.int64)
            im.append(t[0]); om.append(t[1])
        else:
            im.append(np.zeros(0, np.int64)); om.append(np.zeros(0, np.int64))
    return im, om


def oracle_conv_layer(in_coords, tensor_stride, kernel_size, stride, dilation, transposed=False,
                      out_coords=None, region_type=O.HYPER_CUBE):
    """Oracle-side coordinate + kernel-map construction of one (transposed) conv layer.
    Returns (out_coords canonical, in_maps, out_maps)."""
    D = in_coords.shape[1] - 1
    ks, st, dl = [kernel_size] * D, [stride] * D, [dilation] * D
    if not transposed:
        if out_coords is None:
            out_coords, _ = O.stride_map_coords(in_coords, tensor_stride, st)
        offs = O.region_offsets(region_type, ks, dl, tensor_stride)
        im, om = O.kernel_map(in_coords, out_coords, offs)
    else:
        out_ts = [t // s for t, s in zip(tensor_stride, st)]
        assert out_coords is not None
        offs = O.region_offsets(region_type, ks, dl, out_ts)
        im, om = O.transposed_kernel_map(in_coords, out_coords, offs)
    return out_coords, im, om


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def golden(name):
    """A results file of the compiled reference (written by tests/golden/make_reference_runs.py)."""
    return np.load(os.path.join(GOLDEN, name))


def digest(t):
    """SHA-256 of a tensor's values in a fixed dtype per kind (int -> int64, float -> float32)."""
    a = np.ascontiguousarray(np.asarray(t.detach().cpu() if torch.is_tensor(t) else t))
    a = a.astype(np.int64) if a.dtype.kind in "iub" else a.astype(np.float32)
    return np.frombuffer(hashlib.sha256(a.tobytes() + str(a.shape).encode()).digest(), np.uint8)


def state_digest(module):
    """Digest of a module's state_dict (parameters and buffers, in key order)."""
    h = hashlib.sha256()
    for k, v in module.state_dict().items():
        h.update(k.encode())
        h.update(digest(v).tobytes())
    return np.frombuffer(h.digest(), np.uint8)
