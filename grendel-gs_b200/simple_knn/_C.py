"""`from simple_knn._C import distCUDA2` (/root/reference/scene/gaussian_model.py:20,163-166): start-up scale
initialisation only, not on the training path.

CUDA tensors go to the C-ABI search gs_knn3_mean_dist2_range (an exact Morton-tree 3-NN, DESIGN.md 5i) and fail loudly
if the library is missing.  It returns, bit for bit, what the exhaustive kernel gs_knn3_mean_dist2 returns (self
excluded by index, duplicates at distance 0); that kernel stays as the reference the tests compare against
(_dist2_brute; tests/test_point_cloud_gpu.py).  CPU tensors (the reference never passes one: gaussian_model.py:163 calls
`.cuda()` first) get the same definition from exact coordinate differences -- NOT from torch.cdist's |a|^2 + |b|^2 - 2ab
matmul form, which cancels catastrophically in fp32 for near neighbours of an off-origin cloud (every distance of a
3000-point cloud with 2.6e-3 spacing around (30,-20,15) came out 0)."""
import torch


def _dist2_exact_torch(pts):
    """Exact 3-NN mean squared distance from coordinate differences, in chunks; self excluded BY INDEX."""
    n = pts.shape[0]
    out = torch.zeros((n,), dtype=torch.float32, device=pts.device)
    k = min(3, n - 1)
    if k <= 0:
        return out
    chunk = max(1, min(n, (1 << 24) // max(n, 1)))
    cols = torch.arange(n, device=pts.device)
    for s in range(0, n, chunk):
        q = pts[s:s + chunk]
        d = (q[:, None, :] - pts[None, :, :]).square().sum(-1)
        d[torch.arange(q.shape[0], device=pts.device), cols[s:s + chunk]] = float("inf")
        out[s:s + chunk] = d.topk(k, dim=1, largest=False).values.mean(dim=1)
    return out


def _cuda_points(pts):
    if not pts.is_cuda:
        raise TypeError("distCUDA2 kernel path needs a CUDA tensor")
    if pts.dim() != 2 or pts.shape[1] != 3:
        raise ValueError(f"points must be (N, 3), got {tuple(pts.shape)}")
    return pts.float().contiguous()


def _dist2_range(pts, q0, q1):
    """Mean squared distance to the 3 nearest other points of the whole cloud, for points [q0, q1) only: (q1 - q0,)
    float32.  A non-finite coordinate anywhere in the cloud raises ValueError before the search."""
    from gs_b200 import _lib
    pts = _cuda_points(pts)
    n = pts.shape[0]
    if not 0 <= q0 <= q1 <= n:
        raise ValueError(f"query range [{q0}, {q1}) is outside [0, {n}]")
    out = torch.empty((q1 - q0,), dtype=torch.float32, device=pts.device)
    if q0 == q1:
        return out
    with torch.cuda.device(pts.device):   # the library launches on the current device: make it the points' own
        need = _lib.query("gs_knn3_temp_bytes", n)
        if need == 0:
            raise _lib.GsError(f"gs_knn3_temp_bytes failed: {_lib.load().gs_last_error().decode(errors='replace')}")
        temp = torch.empty((need,), dtype=torch.uint8, device=pts.device)
        rc = _lib.query("gs_knn3_mean_dist2_range", n, pts.data_ptr(), q0, q1, out.data_ptr(), temp.data_ptr(),
                        temp.numel(), torch.cuda.current_stream(pts.device).cuda_stream)
    if rc != 0:
        msg = f"gs_knn3_mean_dist2_range failed (code {rc}): {_lib.load().gs_last_error().decode(errors='replace')}"
        raise ValueError(msg) if rc == -1 else _lib.GsError(msg)
    return out


def _dist2_kernel(pts):
    """distCUDA2 of a CUDA tensor: the search over every point."""
    return _dist2_range(pts, 0, pts.shape[0])


def _dist2_brute(pts):
    """The exhaustive O(N^2) kernel: the reference the search is checked against."""
    from gs_b200 import _lib
    pts = _cuda_points(pts)
    out = torch.empty((pts.shape[0],), dtype=torch.float32, device=pts.device)
    with torch.cuda.device(pts.device):
        _lib.call("gs_knn3_mean_dist2", pts.shape[0], pts.data_ptr(), out.data_ptr(),
                  torch.cuda.current_stream(pts.device).cuda_stream)
    return out


def distCUDA2(points):
    """Mean squared distance to the 3 nearest neighbours of every point, (N,) float32."""
    pts = points.float()
    if pts.is_cuda:
        return _dist2_kernel(pts)
    return _dist2_exact_torch(pts)
