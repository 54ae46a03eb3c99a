"""Where does init_data() spend its time?  Wraps the sections of GlobalReconOptimizer.init_data with a synchronising wall-clock
(host + device inclusive per section) and, separately, captures one un-instrumented call with torch.profiler (CUPTI) to list the
device kernels and the device-busy fraction.

    python tools/init_breakdown.py [T=300] [P=1]      env: CFG=glamr_dynamic GAPS=0|1
"""
import copy, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from glamr_b200 import synthetic as syn
from glamr_b200.config import Config
from glamr_b200.recon import GlobalReconOptimizer
from glamr_b200.smpl import SMPL
from glamr_b200.motion_traj import MotionTrajJointModel
from glamr_b200.synthetic_nets import make_prior_states

T = int(sys.argv[1]) if len(sys.argv) > 1 else 300
P = int(sys.argv[2]) if len(sys.argv) > 2 else 1
dev = torch.device('cuda:0')
assets = syn.make_smpl_assets(0)
cfg = Config(os.environ.get('CFG', 'glamr_dynamic'), out_dir='/tmp/e2e')
smpl = SMPL(assets, device=dev)
mt = MotionTrajJointModel(None, dev, None, smpl, make_prior_states())
model = GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=mt)
in_dict = syn.make_in_dict(assets, P, T, seed=0, gaps=os.environ.get('GAPS', '0') == '1')
for _ in range(3):
    model.init_data(copy.deepcopy(in_dict))
torch.cuda.synchronize()

# ---- plain wall clock of the un-instrumented call
ts = []
for _ in range(5):
    d = copy.deepcopy(in_dict)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    model.init_data(d)
    torch.cuda.synchronize()
    ts.append((time.perf_counter() - t0) * 1e3)
print(f'init_data wall ms (P={P}, T={T}): median {np.median(ts):.2f}  all {[round(t, 2) for t in ts]}')

# ---- synchronising section timers
acc = {}


def wrap(obj, name, label=None):
    fn = getattr(obj, name)
    label = label or name

    def timed(*a, **k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*a, **k)
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        e = acc.setdefault(label, [0.0, 0.0, 0])
        e[0] += (t1 - t0) * 1e3
        e[1] += (t2 - t0) * 1e3
        e[2] += 1
        return out
    setattr(obj, name, timed)


for n in ['_persons_from_estimates', '_interp_orient_q_sep_heading', 'infer_motion_traj_all', 'init_cam_pose', 'init_traj_heading_from_cam', '_attach', 'forward', '_take_prior_output']:
    wrap(model, n)
wrap(mt, 'inference', 'mt_model.inference')
REP = 5
for _ in range(REP):
    model.init_data(copy.deepcopy(in_dict))
print(f'{"section":32s} {"host ms":>9s} {"host+device ms":>15s} {"calls":>6s}   (per init_data, sections synchronised; nested sections overlap their parents)')
for k, (h, hd, c) in acc.items():
    print(f'{k:32s} {h / REP:9.3f} {hd / REP:15.3f} {c / REP:6.1f}')

# ---- device kernels of one plain call
for n in list(acc) and []:
    pass
model2 = GlobalReconOptimizer(cfg, dev, None, smpl=smpl, mt_model=MotionTrajJointModel(None, dev, None, smpl, make_prior_states()))
for _ in range(2):
    model2.init_data(copy.deepcopy(in_dict))
torch.cuda.synchronize()
from torch.profiler import profile, ProfilerActivity
d = copy.deepcopy(in_dict)
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    model2.init_data(d)
    torch.cuda.synchronize()
ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
busy = sum(e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total for e in ev)
print(f'device events {len(ev)}, device busy {busy / 1e3:.3f} ms')
agg = {}
for e in ev:
    t = e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
    a = agg.setdefault(e.name[:90], [0, 0.0])
    a[0] += 1
    a[1] += t
for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1])[:30]:
    print(f'{t / 1e3:9.3f} ms {c:5d}  {k}')
print(prof.key_averages().table(sort_by='self_cpu_time_total', row_limit=25, max_name_column_width=60))
