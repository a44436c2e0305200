"""Generate tests/golden/registration_data.npz by running the REFERENCE's own data classes, imported unmodified from
/root/reference/registration, on CPU in this (GPU-less) container.

    python tests/golden/make_registration_data_golden.py

The stubs for kornia and h5py are make_golden.py's; the h5 reading of ModelNetCls is replaced by synthetic clouds
(`_get_data_files` / `_load_data_file` patched, nothing else).  Stored:
  transforms_seed0    QuaternionFixedDataset(197 clouds, repeat=25, seed=0).transforms as (4925, 7) float32 rows
  transforms_seed1    QuaternionFixedDataset(100 clouds, repeat=5, seed=1).transforms as (500, 7)
  clouds              the synthetic set (S, P, 3) float32 as read from the files; num_points the ModelNetCls argument
  perm, p0, p1, vec   QuaternionFixedDataset(ModelNetCls(num_points, OnUnitCube), repeat, seed=0)[r] for every record r: the point
                      permutation ModelNetCls.__getitem__ drew (np.random.seed(1000 + r) before each item, then redrawn the same way), its
                      normalised output p0, the rotated p1 and the transform row

The fixture cannot be regenerated on the GPU box (no reference tree there); it is committed.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/registration"


def main():
    sys.path.insert(0, HERE)
    from make_golden import install_stubs

    install_stubs()
    sys.path.insert(0, REF)
    import data.modelnet_loader_torch as mlt  # noqa: E402  (reference, unmodified)
    from src.pctransforms import OnUnitCube, PointcloudToTensor  # noqa: E402
    from src.qdataset import QuaternionFixedDataset  # noqa: E402

    sets = {}

    def fake_set(num_clouds, num_points_file, seed):
        rng = np.random.default_rng(seed)
        pts = (rng.random((num_clouds, num_points_file, 3), dtype=np.float32) * np.float32(1.6) - np.float32(0.7)).astype(np.float32)
        pts *= np.array([1.0, 0.6, 0.8], np.float32)      # unequal extents: the largest one sets the scale
        sets[seed] = pts
        mlt._get_data_files = lambda _: ["set_%d" % seed]
        mlt._load_data_file = lambda _: (sets[seed], np.zeros((num_clouds, 1), np.int64))
        return pts

    def to_unit_cube(points):   # torchvision.transforms.Compose([PointcloudToTensor(), OnUnitCube()]) of main.py:602
        return OnUnitCube()(PointcloudToTensor()(points))

    def table(num_clouds, repeat, seed):
        fake_set(num_clouds, 8, 50 + num_clouds)
        base = mlt.ModelNetCls(8, transforms=to_unit_cube, train=True, download=False, folder="none")
        qds = QuaternionFixedDataset(base, repeat=repeat, seed=seed)
        return torch.cat([t.vec for t in qds.transforms]).numpy()

    out = {"transforms_seed0": table(197, 25, 0), "transforms_seed1": table(100, 5, 1)}

    S, P, num_points, repeat = 3, 300, 256, 2
    clouds = fake_set(S, P, 7)
    base = mlt.ModelNetCls(num_points, transforms=to_unit_cube, train=True, download=False, folder="none")
    qds = QuaternionFixedDataset(base, repeat=repeat, seed=0)
    perm, p0, p1, vec = [], [], [], []
    for r in range(len(qds)):
        np.random.seed(1000 + r)
        a, b, igt = qds[r]
        np.random.seed(1000 + r)
        idx = np.arange(0, num_points)
        np.random.shuffle(idx)
        perm.append(idx.astype(np.int32))
        p0.append(a.numpy())
        p1.append(b.numpy())
        vec.append(igt["vec"].numpy()[0])
    np.savez_compressed(os.path.join(HERE, "registration_data.npz"), clouds=clouds, num_points=np.int32(num_points), repeat=np.int32(repeat),
                        perm=np.stack(perm), p0=np.stack(p0), p1=np.stack(p1), vec=np.stack(vec), **out)
    print("registration_data.npz written to", HERE)


if __name__ == "__main__":
    main()
