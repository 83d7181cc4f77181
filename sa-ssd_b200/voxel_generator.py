"""VoxelGenerator — mmdet/core/point_cloud/voxel_generator.py:4-43 over the CUDA
voxelizer (csrc/voxelize.cu) instead of the numba loop (points_ops.py:104-164)."""
import numpy as np
import torch

from . import ops


class VoxelGenerator:
    """Constructor kwargs as in configs/car_cfg.py:116-122."""

    def __init__(self, voxel_size, point_cloud_range, max_num_points, max_voxels=20000, device="cuda"):
        self._point_cloud_range = np.array(point_cloud_range, dtype=np.float32)
        self._voxel_size = np.array(voxel_size, dtype=np.float32)
        self._max_num_points = int(max_num_points)
        self._max_voxels = int(max_voxels)
        self._params, grid = ops.make_voxel_params(self._voxel_size, self._point_cloud_range, max_num_points,
                                                   max_voxels)
        self._grid_size = grid
        self.device = device

    @property
    def voxel_size(self):
        return self._voxel_size

    @property
    def max_num_points_per_voxel(self):
        return self._max_num_points

    @property
    def max_voxels(self):
        return self._max_voxels

    @property
    def point_cloud_range(self):
        return self._point_cloud_range

    @property
    def grid_size(self):
        return self._grid_size

    def generate_device(self, points, pt_off, batch, max_points_per_frame, status, rows_cap=None):
        """points [Ncap,4] device, pt_off [batch+1] int32 device.  No sync.  Returns
        (voxels [cap,P,4], coors [cap,4] (b,z,y,x), num_points [cap], mean [cap,4], frame_rows [batch+1])."""
        slots = ops.next_pow2(2 * max(int(max_points_per_frame), 1))
        if rows_cap is None:
            rows_cap = batch * min(self._max_voxels, max(int(max_points_per_frame), 1))
        return ops.voxelize(points, pt_off, batch, self._params, max(rows_cap, 1), slots, status)

    def generate(self, points):
        """Reference API: points [N,>=4] numpy -> (voxels [M,P,4], coordinates [M,3] (z,y,x), num_points [M])."""
        ops.require_cuda()
        pts = np.ascontiguousarray(points[:, :4], dtype=np.float32)
        n = pts.shape[0]
        dev = torch.device(self.device)
        d_pts = torch.from_numpy(pts).to(dev) if n else torch.zeros((1, 4), dtype=torch.float32, device=dev)
        pt_off = torch.tensor([0, n], dtype=torch.int32, device=dev)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        voxels, coors, num, _, frame_rows = self.generate_device(d_pts, pt_off, 1, n, status)
        m = int(frame_rows[1].item())
        ops._lib.raise_on_status(status)
        return (voxels[:m].cpu().numpy(), coors[:m, 1:].contiguous().cpu().numpy(), num[:m].cpu().numpy())
