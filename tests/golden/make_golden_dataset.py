#!/usr/bin/env python
"""Golden items of the input side (DESIGN 3.19), written by the REFERENCE'S OWN `pointmvsnet/dataset.py` and
`utils/preprocess.py` (imported from the reference checkout at REF, nothing copied) on a synthetic DTU tree this
script builds: `Cameras/pair.txt` with 3 views, camera texts, PNG views and PFM depth maps.  `dataset_small.npz` holds
the tree's inputs and the reference's outputs: the path lists of the train, valid and test sets, one train item, and
one test item with and without `depth_folder`.  `build_tree(root, z)` rebuilds the same tree from the npz.

Test geometry: raw 240 x 180 views with IMG_HEIGHT 128 and IMG_WIDTH 192, so the resize factor is 0.8 (144 x 192),
the crop removes 8 rows and the 1/8 grid is 16 x 24; the test depth maps are 60 x 80.  The depth maps hold values
at, and one float32 ulp either side of, both masking thresholds, and an infinity.

Adjustments, applied from outside, for a current install: `tqdm` (not a dependency of this project) is stubbed, and
`np.float` (removed in numpy 2, dataset.py:265) is restored as an alias of the builtin.
"""
import os
import sys
import tempfile
import types

import cv2
import numpy as np
import torch

REF = "/root/reference"
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from pointmvsnet_b200.utils.io import write_pfm  # noqa: E402

NUM_VIEW = 3
TRAIN_HW = (48, 64)
TEST_HW = (180, 240)
TEST_OUT = (128, 192)
NUM_PLANE = 48
INTERVAL_SCALE = 1.6


def pair_text():
    rows = ["%d" % NUM_VIEW]
    for i in range(NUM_VIEW):
        others = [(i + 1 + k) % NUM_VIEW for k in range(10)]
        others = [o if o != i else (o + 1) % NUM_VIEW for o in others]
        rows.append("%d" % i)
        rows.append("10 " + " ".join("%d %.4f" % (o, 100.0 - k) for k, o in enumerate(others)))
    return "\n".join(rows) + "\n"


def cam_text(i, f, cx, cy):
    rot = [[1.0, 0.0, 0.0], [0.0, 1.0, 0.0], [0.0, 0.0, 1.0]]
    t = [-10.0 * i, 2.5 * i, 0.5]
    rows = ["extrinsic"]
    for r in range(3):
        rows.append(" ".join("%.6f" % v for v in rot[r] + [t[r]]))
    rows += ["0.0 0.0 0.0 1.0", "", "intrinsic", "%.4f 0.0 %.4f" % (f, cx), "0.0 %.4f %.4f" % (f, cy),
             "0.0 0.0 1.0", "", "%.3f %.3f" % (425.0 + 3.0 * i, 2.5)]
    return "\n".join(rows) + "\n"


def image(g, h, w):
    """smooth BGR gradients plus noise, uint8"""
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64),
                            indexing="ij")
    base = torch.stack([128 + 90 * torch.sin(xx / 17 + c) * torch.cos(yy / 23 - c) for c in range(3)], -1)
    return (base + 20 * torch.randn(h, w, 3, generator=g, dtype=torch.float64)).round().clamp(0, 255).to(
        torch.uint8).numpy()


def depth(g, h, w, start, end):
    """depths in (start - 20, end + 20) with the float32 neighbours of both thresholds and an infinity planted"""
    d = (start - 20 + (end - start + 40) * torch.rand(h, w, generator=g, dtype=torch.float64)).numpy()
    d = (np.round(d * 4) / 4).astype(np.float32)  # quarter steps: the file compresses
    special = []
    for t in (np.float32(start), np.float32(end)):
        special += [np.nextafter(t, np.float32(-np.inf)), t, np.nextafter(t, np.float32(np.inf))]
    special += [np.float32(np.inf), np.float32(0)]
    for k, v in enumerate(special):
        d[k % h, (3 * k) % w] = v
    return d


def make_inputs():
    g = torch.Generator().manual_seed(11)
    z = {"pair_txt": np.array(pair_text())}
    for i in range(NUM_VIEW):
        z["cam_train_%d" % i] = np.array(cam_text(i, 57.7 + i, 31.5 + 0.25 * i, 23.5 - 0.5 * i))
        z["cam_test_%d" % i] = np.array(cam_text(i, 361.54 + i, 119.5 + 0.5 * i, 89.5 - 0.25 * i))
        z["img_train_%d" % i] = image(g, *TRAIN_HW)
        z["img_test_%d" % i] = image(g, *TEST_HW)
        start0 = 425.0 + 2.5 * INTERVAL_SCALE  # view 0's depth_min + interval
        end0 = 425.0 + (NUM_PLANE - 2) * 2.5 * INTERVAL_SCALE
        z["depth_train_%d" % i] = depth(g, TRAIN_HW[0] // 4, TRAIN_HW[1] // 4, start0, end0)
        z["depth_test_%d" % i] = depth(g, TEST_HW[0] // 3, TEST_HW[1] // 3, start0, end0)
    return z


def build_tree(root, z):
    """write the synthetic scan tree of `z` (make_inputs() or the npz) under root; -> the depth folder"""
    def put(path, text):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as f:
            f.write(str(text))

    def put_png(path, img):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        assert cv2.imwrite(path, np.asarray(img))

    def put_pfm(path, d):
        os.makedirs(os.path.dirname(path), exist_ok=True)
        write_pfm(path, np.asarray(d, np.float32))

    depth_folder = os.path.join(root, "depths_out")
    put(os.path.join(root, "Cameras", "pair.txt"), z["pair_txt"])
    for i in range(NUM_VIEW):
        put(os.path.join(root, "Cameras", "train", "%08d_cam.txt" % i), z["cam_train_%d" % i])
        put(os.path.join(root, "Cameras", "%08d_cam.txt" % i), z["cam_test_%d" % i])
        put_png(os.path.join(root, "Rectified", "scan2_train", "rect_%03d_0_r5000.png" % (i + 1)),
                z["img_train_%d" % i])
        put_pfm(os.path.join(root, "Depths", "scan2_train", "depth_map_%04d.pfm" % i), z["depth_train_%d" % i])
        put_png(os.path.join(root, "Eval", "Rectified", "scan1", "rect_%03d_3_r5000.png" % (i + 1)),
                z["img_test_%d" % i])
        put_pfm(os.path.join(depth_folder, "scan1", "depth_map_%04d.pfm" % i), z["depth_test_%d" % i])
    return depth_folder


def path_array(path_list, root, depth_folder):
    """[entries, 3, V] strings with the tree's root as <root> and the depth folder as <depth>"""
    def rel(p):
        return p.replace(depth_folder, "<depth>").replace(root, "<root>")
    return np.array([[[rel(p) for p in e[k]] for k in ("view_image_paths", "view_cam_paths", "view_depth_paths")]
                     for e in path_list])


def main():
    sys.path.insert(0, REF)
    sys.modules["tqdm"] = types.SimpleNamespace(tqdm=lambda x, *a, **k: x)  # see module docstring
    np.float = float
    from pointmvsnet import dataset as ref

    z = make_inputs()
    out = dict(z)
    with tempfile.TemporaryDirectory() as root:
        depth_folder = build_tree(root, z)
        train = ref.DTU_Train_Val_Set(root, "train", num_view=NUM_VIEW, num_virtual_plane=NUM_PLANE,
                                      interval_scale=INTERVAL_SCALE)
        valid = ref.DTU_Train_Val_Set(root, "valid", num_view=NUM_VIEW, num_virtual_plane=NUM_PLANE,
                                      interval_scale=INTERVAL_SCALE)
        kw = dict(num_view=NUM_VIEW, height=TEST_OUT[0], width=TEST_OUT[1], num_virtual_plane=NUM_PLANE,
                  interval_scale=INTERVAL_SCALE)
        test = ref.DTU_Test_Set(root, "test", depth_folder=depth_folder, **kw)
        test_nd = ref.DTU_Test_Set(root, "test", **kw)
        out["paths_train"] = path_array(train.path_list, root, depth_folder)
        out["paths_valid"] = path_array(valid.path_list, root, depth_folder)
        out["paths_test"] = path_array(test.path_list, root, depth_folder)
        out["paths_test_nodepth"] = path_array(test_nd.path_list, root, depth_folder)
        for name, ds in (("train", train), ("test", test), ("test_nodepth", test_nd)):
            item = ds[0]
            for k, v in item.items():
                if k == "ref_img_path":
                    v = np.array(v.replace(root, "<root>"))
                elif k == "img_list" and name == "test_nodepth":
                    assert torch.equal(v, out["test_img_list"]), "img_list does not depend on depth_folder"
                    continue
                elif isinstance(v, torch.Tensor):
                    v = v.numpy()
                out["%s_%s" % (name, k)] = v
                if name == "test" and k == "img_list":
                    out["test_img_list"] = torch.from_numpy(v)
        out["test_img_list"] = out["test_img_list"].numpy()
    np.savez_compressed(os.path.join(HERE, "dataset_small.npz"), **out)
    print("wrote dataset_small.npz:", {k: getattr(v, "shape", None) for k, v in out.items() if "paths" not in k})


if __name__ == "__main__":
    main()
