import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointmvsnet_b200 import _lib
from pointmvsnet_b200.cost_volume import build_cost_volume
from pointmvsnet_b200.synthetic import make_cameras
dev = torch.device("cuda:0")
feats = torch.randn(1, 4, 64, 64, 80, device=dev); cams = make_cameras(1, 4, 512, 640, 96).to(dev)
for _ in range(3): c = build_cost_volume(feats, cams)
torch.cuda.synchronize(); _lib.profile_enable(True)
for _ in range(5): c = build_cost_volume(feats, cams)
torch.cuda.synchronize(); _lib.profile_enable(False)
r = [ms for n, ms in _lib.profile_collect() if n == "cost_volume"]
gb = (4 * 64 * 64 * 80 * 4 + 64 * 96 * 64 * 80 * 4) / 1e9
print("cost_volume C2: %.1f us, %.0f GB/s algorithmic" % (1e3 * sum(r) / len(r), gb / (sum(r) / len(r) * 1e-3)))
