"""BASELINE config 3: motion_infiller + traj_pred inference, batch 64 x 120-frame sequences, 1 GPU (ms per batch)."""
import os, sys, time, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from glamr_b200.motion_traj import MotionTrajJointModel
from glamr_b200.smpl import SMPL
from glamr_b200.synthetic import make_smpl_assets
from glamr_b200.synthetic_nets import make_prior_states
B, T = int(os.environ.get('B', 64)), int(os.environ.get('T', 120))
dev = torch.device('cuda:0')
m = MotionTrajJointModel(None, dev, None, smpl=SMPL(make_smpl_assets(0), device=dev), states=make_prior_states(1234))
g = torch.Generator().manual_seed(0)
pose = (torch.randn(B, T, 69, generator=g) * 0.3).to(dev); mask = torch.ones(B, T, device=dev); mask[:, 40:70] = 0
nw = -(-(T - 10) // 30)
batch = {'in_body_pose': pose * mask[..., None], 'frame_mask': mask, 'in_motion_latent': torch.randn(nw, 128, generator=g).to(dev), 'in_traj_latent': torch.randn(1, 128, generator=g).to(dev)}
for _ in range(3): m.inference(batch)
torch.cuda.synchronize(); t0 = time.perf_counter()
for _ in range(10): m.inference(batch)
torch.cuda.synchronize()
print(f'B={B} T={T}: {(time.perf_counter() - t0) / 10 * 1e3:.2f} ms/batch')
