"""The DTU loaders (the reference's pointmvsnet/dataset.py), with the pixel work on the device (DESIGN 3.19).

`DTU_Train_Val_Set` and `DTU_Test_Set` take the reference's constructor arguments and walk the same scan and lighting
lists, `Cameras/pair.txt` entries and file names.  Their items are what a DataLoader worker produces: the 8-bit views
as cv2.imread returns them, cameras scaled and cropped on the host in float64 and cast to float32, and the depth maps
masked on the host.  Workers never touch CUDA.  `build_data_loader(cfg, mode)` wraps the dataset in a `DeviceLoader`:
iterating it copies each pinned batch to the current CUDA device and runs `prepare_views` there, and yields the dict
the reference's `__getitem__` + `default_collate` + `.cuda()` would give, with the same keys, shapes and dtypes.  So
train.py / test.py, `PointMVSNet`, `PointMVSNetLoss` and `eval_file_logger` take it unchanged.

`img_list` is normalised with the exact per-view statistics, not numpy's float32 accumulation (DESIGN 3.19).
"""
import os.path as osp

import cv2
import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

from .utils import io
from .utils.preprocess import (crop_geometry, mask_depth_image, prepare_views, resize_factor, resized_size,
                               scale_camera, shift_camera)

__all__ = ["DTU_Train_Val_Set", "DTU_Test_Set", "DeviceLoader", "build_data_loader"]

MEAN = (1.97145182, -1.52387525, 651.07223895)
STD = (84.45612252, 93.22252387, 80.08551226)
PAIR_TOKENS = 22  # per reference view in pair.txt: its index, the count 10, then 10 (index, score) pairs


def _read_pairs(root_dir, cluster_file_path):
    with open(osp.join(root_dir, cluster_file_path)) as f:
        return f.read().split()


def _walk(cluster_list, num_view, scans, lightings, image_folder, cam_folder, depth_folder):
    """one entry per (scan, lighting, reference view): the image, camera and depth paths of the reference view and
    its first num_view - 1 source views, in pair.txt order"""
    out = []
    for scan in scans:
        img_dir, depth_dir = image_folder(scan), depth_folder(scan)
        for light in lightings:
            for p in range(int(cluster_list[0])):
                base = PAIR_TOKENS * p
                views = [int(cluster_list[base + 1])] + [int(cluster_list[base + 2 * v + 3])
                                                         for v in range(num_view - 1)]
                out.append({
                    "view_image_paths": [osp.join(img_dir, "rect_{:03d}_{}_r5000.png".format(i + 1, light))
                                         for i in views],
                    "view_cam_paths": [osp.join(cam_folder, "{:08d}_cam.txt".format(i)) for i in views],
                    "view_depth_paths": [osp.join(depth_dir, "depth_map_{:04d}.pfm".format(i)) for i in views],
                })
    return out


def _read_views(paths):
    """uint8 [V, H0, W0, 3] BGR; views of different sizes raise here, before anything is copied"""
    images = []
    for p in paths:
        img = cv2.imread(p)
        if img is None:
            raise FileNotFoundError("cannot read image %s" % p)
        if images and img.shape != images[0].shape:
            raise ValueError("views of one sample differ in size: %s is %s, %s is %s"
                             % (paths[0], images[0].shape, p, img.shape))
        images.append(img)
    return np.stack(images)


def _read_cams(paths, num_depth, interval_scale):
    cams = []
    for p in paths:
        with open(p) as f:
            cams.append(io.load_cam_dtu(f, num_depth=num_depth, interval_scale=interval_scale))
    return cams


def _geometry(scale, y0, x0, h, w):
    return torch.tensor([scale, y0, x0, h, w], dtype=torch.float64)


class DTU_Train_Val_Set(Dataset):
    training_set = [2, 6, 7, 8, 14, 16, 18, 19, 20, 22, 30, 31, 36, 39, 41, 42, 44,
                    45, 46, 47, 50, 51, 52, 53, 55, 57, 58, 60, 61, 63, 64, 65, 68, 69, 70, 71, 72,
                    74, 76, 83, 84, 85, 87, 88, 89, 90, 91, 92, 93, 94, 95, 96, 97, 98, 99, 100,
                    101, 102, 103, 104, 105, 107, 108, 109, 111, 112, 113, 115, 116, 119, 120,
                    121, 122, 123, 124, 125, 126, 127, 128]
    validation_set = [3, 5, 17, 21, 28, 35, 37, 38, 40, 43, 56, 59, 66, 67, 82, 86, 106, 117]
    training_lighting_set = [0, 1, 2, 3, 4, 5, 6]
    validation_lighting_set = [3]
    mean = torch.tensor(MEAN)
    std = torch.tensor(STD)
    cluster_file_path = "Cameras/pair.txt"

    def __init__(self, root_dir, dataset_name, num_view=3, num_virtual_plane=128, interval_scale=1.6):
        self.root_dir = root_dir
        self.num_view = num_view
        self.interval_scale = interval_scale
        self.num_virtual_plane = num_virtual_plane
        self.cluster_list = _read_pairs(root_dir, self.cluster_file_path)
        # "val" is the name build_data_loader(cfg, "val") passes; the reference's assert rejected it, so its
        # validation loop could never start.  Here it serves the validation set, as "valid" does.
        if dataset_name == "train":
            self.data_set, self.lighting_set = self.training_set, self.training_lighting_set
        elif dataset_name in ("valid", "val"):
            self.data_set, self.lighting_set = self.validation_set, self.validation_lighting_set
        else:
            raise ValueError("Unknown dataset_name: {}".format(dataset_name))
        self.path_list = _walk(self.cluster_list, num_view, self.data_set, self.lighting_set,
                               lambda s: osp.join(root_dir, "Rectified/scan{}_train".format(s)),
                               osp.join(root_dir, "Cameras/train"),
                               lambda s: osp.join(root_dir, "Depths/scan{}_train".format(s)))

    def __getitem__(self, index):
        paths = self.path_list[index]
        views = _read_views(paths["view_image_paths"][:self.num_view])
        cams = _read_cams(paths["view_cam_paths"][:self.num_view], self.num_virtual_plane, self.interval_scale)
        depths = [io.load_pfm(p)[0] for p in paths["view_depth_paths"]]

        depth_start = cams[0][1, 3, 0] + cams[0][1, 3, 1]
        depth_end = cams[0][1, 3, 0] + (self.num_virtual_plane - 2) * cams[0][1, 3, 1]
        ref_depth = mask_depth_image(depths[0], depth_start, depth_end)
        depth_list = torch.tensor(np.stack(depths)).unsqueeze(1).float()
        # the reference's arithmetic: an infinite depth times a zero mask is NaN
        depth_list = depth_list * (depth_list > depth_start).float() * (depth_list < depth_end).float()
        return {
            "views": torch.from_numpy(views),
            "geometry": _geometry(1.0, 0, 0, views.shape[1], views.shape[2]),
            "cam_params_list": torch.tensor(np.stack(cams)).float(),
            "gt_depth_img": torch.tensor(ref_depth).permute(2, 0, 1).float(),
            "depth_list": depth_list,
            "ref_img_path": paths["view_image_paths"][0],
            "mean": self.mean,
            "std": self.std,
        }

    def __len__(self):
        return len(self.path_list)


class DTU_Test_Set(Dataset):
    test_set = [1, 4, 9, 10, 11, 12, 13, 15, 23, 24, 29, 32, 33, 34, 48, 49, 62, 75, 77,
                110, 114, 118]
    test_lighting_set = [3]
    mean = torch.tensor(MEAN)
    std = torch.tensor(STD)
    cluster_file_path = "Cameras/pair.txt"

    def __init__(self, root_dir, dataset_name, num_view=3, height=1152, width=1600, num_virtual_plane=128,
                 interval_scale=1.6, base_image_size=64, depth_folder=""):
        self.root_dir = root_dir
        self.num_view = num_view
        self.interval_scale = interval_scale
        self.num_virtual_plane = num_virtual_plane
        self.base_image_size = base_image_size
        self.height = height
        self.width = width
        self.depth_folder = depth_folder
        self.cluster_list = _read_pairs(root_dir, self.cluster_file_path)
        if dataset_name != "test":
            raise ValueError("Unknown dataset_name: {}".format(dataset_name))
        self.data_set, self.lighting_set = self.test_set, self.test_lighting_set
        self.path_list = _walk(self.cluster_list, num_view, self.data_set, self.lighting_set,
                               lambda s: osp.join(root_dir, "Eval/Rectified/scan{}".format(s)),
                               osp.join(root_dir, "Cameras"),
                               lambda s: osp.join(depth_folder, "scan{}".format(s)))

    def __getitem__(self, index):
        paths = self.path_list[index]
        views = _read_views(paths["view_image_paths"][:self.num_view])
        cams = _read_cams(paths["view_cam_paths"][:self.num_view], self.num_virtual_plane, self.interval_scale)
        if self.depth_folder:
            depths = [io.load_pfm(p)[0] for p in paths["view_depth_paths"]]
        else:  # float64 zeros of the requested size, as the reference makes them
            depths = [np.zeros((self.height, self.width), np.float64) for _ in paths["view_depth_paths"]]

        h0, w0 = views.shape[1:3]
        scale = resize_factor(h0, w0, self.height, self.width)
        h, w = resized_size(h0, w0, scale)
        y0, x0, hc, wc = crop_geometry(h, w, self.height, self.width, self.base_image_size)
        cams = [shift_camera(scale_camera(c, scale), y0, x0) for c in cams]
        ref_depth = cv2.resize(depths[0], None, fx=scale, fy=scale, interpolation=cv2.INTER_NEAREST)
        ref_depth = np.ascontiguousarray(ref_depth[y0:y0 + hc, x0:x0 + wc])
        return {
            "views": torch.from_numpy(views),
            "geometry": _geometry(scale, y0, x0, hc, wc),
            "cam_params_list": torch.tensor(np.stack(cams)).float(),
            "gt_depth_img": torch.from_numpy(ref_depth),
            "depth_list": torch.tensor(np.stack(depths)).unsqueeze(1).float(),
            "ref_img_path": paths["view_image_paths"][0],
            "mean": self.mean,
            "std": self.std,
        }

    def __len__(self):
        return len(self.path_list)


class DeviceLoader:
    """A DataLoader (pinned host batches) whose batches come out prepared on the current CUDA device, in the
    reference's dict: the views are copied as uint8 and resized, cropped and normalised by `prepare_views`."""

    def __init__(self, dataset, batch_size, shuffle=False, num_workers=0):
        self.dataset = dataset
        self.test = isinstance(dataset, DTU_Test_Set)
        self.loader = DataLoader(dataset, batch_size, shuffle=shuffle, num_workers=num_workers, pin_memory=True)

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        for batch in self.loader:
            yield self.prepare(batch)

    def prepare(self, batch):
        """a collated host batch of this dataset -> the reference's dict on the current CUDA device"""
        geo = batch["geometry"]
        if not bool((geo == geo[0]).all()):
            raise ValueError("the samples of one batch need the same resize and crop, got %s" % geo.tolist())
        scale, y0, x0, h, w = geo[0].tolist()
        dev = torch.device("cuda", torch.cuda.current_device())
        views = batch["views"].to(dev, non_blocking=True)

        def put(key):
            return batch[key].to(dev, non_blocking=True)

        out = {}
        prepared = prepare_views(views, scale, (int(y0), int(x0)), (int(h), int(w)), ref_image=self.test)
        out["img_list"] = prepared[0] if self.test else prepared
        for key in ("cam_params_list", "gt_depth_img", "depth_list"):
            out[key] = put(key)
        out["ref_img_path"] = batch["ref_img_path"]
        if self.test:
            out["ref_img"] = prepared[1]
        out["mean"] = put("mean")
        out["std"] = put("std")
        return out


def build_data_loader(cfg, mode="train"):
    """the reference's build_data_loader over the same cfg fields (any object with those attributes)"""
    if mode == "train":
        dataset = DTU_Train_Val_Set(root_dir=cfg.DATA.TRAIN.ROOT_DIR, dataset_name="train",
                                    num_view=cfg.DATA.TRAIN.NUM_VIEW, interval_scale=cfg.DATA.TRAIN.INTER_SCALE,
                                    num_virtual_plane=cfg.DATA.TRAIN.NUM_VIRTUAL_PLANE)
    elif mode == "val":
        dataset = DTU_Train_Val_Set(root_dir=cfg.DATA.VAL.ROOT_DIR, dataset_name="val",
                                    num_view=cfg.DATA.VAL.NUM_VIEW, interval_scale=cfg.DATA.TRAIN.INTER_SCALE,
                                    num_virtual_plane=cfg.DATA.TRAIN.NUM_VIRTUAL_PLANE)
    elif mode == "test":
        dataset = DTU_Test_Set(root_dir=cfg.DATA.TEST.ROOT_DIR, dataset_name="test", num_view=cfg.DATA.TEST.NUM_VIEW,
                               height=cfg.DATA.TEST.IMG_HEIGHT, width=cfg.DATA.TEST.IMG_WIDTH,
                               interval_scale=cfg.DATA.TEST.INTER_SCALE,
                               num_virtual_plane=cfg.DATA.TEST.NUM_VIRTUAL_PLANE)
    else:
        raise ValueError("Unknown mode: {}.".format(mode))
    batch_size = cfg.TRAIN.BATCH_SIZE if mode == "train" else cfg.TEST.BATCH_SIZE
    return DeviceLoader(dataset, batch_size, shuffle=(mode == "train"), num_workers=cfg.DATA.NUM_WORKERS)
