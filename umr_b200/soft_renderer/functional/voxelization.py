"""`voxelization` of the drop-in package (reference: SoftRas/functional/voxelization.py) on the csrc/voxel.cu kernels."""
from ... import ops


def voxelization(faces, size, normalize=False):
    """faces [B,F,3,3] (float32 or float64, cuda) -> int32 [B,size,size,size]: surface voxels plus every enclosed empty
    voxel.  Coordinates are multiplied by `size` unless `normalize`.  `faces` is not modified."""
    return ops.voxelize(faces, size, normalize)
