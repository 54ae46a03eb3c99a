"""Sequence sweep: the part of the reference's ``global_recon/run_dataset.py:60-112`` / ``run_demo.py:55-82`` that sits
on the hot path -- ``pose.pkl`` (or a synthetic HybrIK-shaped estimate) -> ``GlobalReconOptimizer.optimize`` ->
``<out_dir>/<seq>/grecon/<seq>_seed<seed>.pkl``, same file naming and pickle layout as the reference.

Pose estimation (HybrIK), visualisation and evaluation are out of scope (SURVEY.md §8): a sequence needs its
``pose.pkl`` on disk (``<pose_root>/<seq>/pose_est/pose.pkl`` as ``run_pose_est_on_video`` leaves it, or
``<pose_root>/<seq>.pkl``), or ``--synthetic N`` generates N seeded sequences.

Independent sequences are replicas (SURVEY.md §8e, BASELINE config 5): under ``torchrun`` rank r takes sequences
r, r + world, ... on its own GPU; there is no collective on the data path.

``--batch_seeds`` optimises the seeds of a sequence together, one ``optimize_seeds`` call per sequence instead of one
``optimize`` call per seed: same files, same contents; each seed's recorded time is the call's time divided by the number of
seeds it ran.

``--batch_sequences K`` optimises a rank's sequences K at a time as the groups of one ``optimize_batch`` call: all remaining
seeds of those sequences with ``--batch_seeds``, one seed per call otherwise.  Same files, same contents; each (sequence, seed)
pair's recorded time is the call's time divided by the number of pairs it ran.  The GPU scratch grows with the frame-persons of
the call (sum of persons x frames over its pairs): about 350 MB at 4,000 frame-persons, mostly the SMPL vertices.

    python -m glamr_b200.global_recon.run_dataset --cfg glamr_3dpw --synthetic 32 --frames 300 --out_dir out/sweep
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 -m glamr_b200.global_recon.run_dataset ...
"""
import argparse
import os
import pickle
import time

import numpy as np


def shard(items, rank, world):
    """round-robin assignment of independent sequences to ranks"""
    return list(items)[rank::world]


def out_file_of(out_dir, seq_name, seed):
    """run_dataset.py:93 / run_demo.py:74"""
    return os.path.join(out_dir, seq_name, 'grecon', f'{seq_name}_seed{seed}.pkl')


def find_pose_file(pose_root, seq_name):
    for cand in (os.path.join(pose_root, seq_name, 'pose_est', 'pose.pkl'), os.path.join(pose_root, f'{seq_name}.pkl')):
        if os.path.exists(cand):
            return cand
    raise FileNotFoundError(f'no pose.pkl for sequence {seq_name} under {pose_root}: pose estimation is not part of glamr_b200')


def load_in_dict(pose_file, seq_name, gt_file=None):
    """run_dataset.py:95-100: est dict (+ optional ground truth) -> the optimiser's in_dict"""
    with open(pose_file, 'rb') as f:
        est = pickle.load(f)
    if gt_file is None:
        return {'est': est, 'gt': dict(), 'gt_meta': dict(), 'seq_name': seq_name}
    with open(gt_file, 'rb') as f:
        gt = pickle.load(f)
    return {'est': est, 'gt': gt['person_data'], 'gt_meta': gt['meta'], 'seq_name': seq_name}


def list_sequences(args):
    if args.synthetic > 0:
        return [f'synthetic_{i:04d}' for i in range(args.synthetic)]
    if args.sequences:
        return args.sequences.split(',')
    names = set()
    for e in sorted(os.listdir(args.pose_root)):
        p = os.path.join(args.pose_root, e)
        if os.path.isdir(p) and os.path.exists(os.path.join(p, 'pose_est', 'pose.pkl')):
            names.add(e)
        elif e.endswith('.pkl'):
            names.add(e[:-4])
    return sorted(names)


def run(args, make_model=None, make_in_dict=None):
    """-> list of (seq_name, seed, out_file, seconds) processed by this rank.  `make_model(cfg, device)` /
    `make_in_dict(seq_name)` are injection points for tests."""
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', args.gpu))
    from glamr_b200.config import Config
    cfg = Config(args.cfg, out_dir=args.out_dir)
    if make_model is None:
        import torch
        from glamr_b200.global_recon.models import model_dict
        device = torch.device('cuda', local)
        torch.cuda.set_device(device)
        smpl, mt = None, None
        if args.synthetic > 0 and not args.real_assets:           # no SMPL model files / checkpoints offline: seeded stand-ins
            from glamr_b200.motion_traj import MotionTrajJointModel
            from glamr_b200.smpl import SMPL
            from glamr_b200.synthetic import make_smpl_assets
            from glamr_b200.synthetic_nets import make_prior_states
            smpl = SMPL(make_smpl_assets(0), device=device)
            if cfg.grecon_model_specs.get('flag_infer_motion_traj', False):      # no learned prior without it
                mt = MotionTrajJointModel(None, device, None, smpl=smpl, states=make_prior_states(1234))
        model = model_dict[cfg.grecon_model_name](cfg, device, None, smpl=smpl, mt_model=mt)
    else:
        model = make_model(cfg, local)
    if make_in_dict is None and args.synthetic > 0:
        from glamr_b200.synthetic import make_in_dict as synth, make_smpl_assets
        assets = make_smpl_assets(0)

        def make_in_dict(seq_name):
            i = int(seq_name.rsplit('_', 1)[1])
            return synth(assets, args.persons, args.frames, seed=i, gaps=args.gaps, seq_name=seq_name)
    seeds = [int(x) for x in str(args.seeds).split(',')]
    done = []
    mine = shard(list_sequences(args), rank, world)
    def load(seq_name):
        if make_in_dict is not None:
            return make_in_dict(seq_name)
        gt_file = os.path.join(args.gt_pose_root, f'{seq_name}.pkl') if args.gt_pose_root else None
        return load_in_dict(find_pose_file(args.pose_root, seq_name), seq_name, gt_file)

    if args.batch_sequences > 0:
        return done + _run_batches(args, model, mine, seeds, load, rank)
    for i, seq_name in enumerate(mine):
        if args.batch_seeds:
            todo = []
            for seed in seeds:
                out_file = out_file_of(args.out_dir, seq_name, seed)
                if args.cached and os.path.exists(out_file):
                    done.append((seq_name, seed, out_file, 0.0))
                else:
                    todo.append((seed, out_file))
            if not todo:
                continue
            in_dict = load(seq_name)
            t0 = time.perf_counter()
            outs = model.optimize_seeds(in_dict, [seed for seed, _ in todo])       # sets the RNGs of every seed itself
            dt = (time.perf_counter() - t0) / len(todo)
            for (seed, out_file), out_dict in zip(todo, outs):
                os.makedirs(os.path.dirname(out_file), exist_ok=True)
                with open(out_file, 'wb') as f:
                    pickle.dump(out_dict, f)
                done.append((seq_name, seed, out_file, dt))
                if not args.quiet:
                    print(f'[rank {rank}] {i + 1}/{len(mine)} seed {seed} {seq_name}: {dt * 1e3:.1f} ms (batch of {len(todo)}) -> {out_file}',
                          flush=True)
            continue
        for seed in seeds:
            out_file = out_file_of(args.out_dir, seq_name, seed)
            if args.cached and os.path.exists(out_file):
                done.append((seq_name, seed, out_file, 0.0))
                continue
            os.makedirs(os.path.dirname(out_file), exist_ok=True)
            np.random.seed(seed)
            try:
                import torch
                torch.manual_seed(seed)
            except ImportError:
                pass
            in_dict = load(seq_name)
            t0 = time.perf_counter()
            out_dict = model.optimize(in_dict)
            dt = time.perf_counter() - t0
            with open(out_file, 'wb') as f:
                pickle.dump(out_dict, f)
            done.append((seq_name, seed, out_file, dt))
            if not args.quiet:
                print(f'[rank {rank}] {i + 1}/{len(mine)} seed {seed} {seq_name}: {dt * 1e3:.1f} ms -> {out_file}', flush=True)
    return done


def _run_batches(args, model, mine, seeds, load, rank):
    """--batch_sequences: the rank's sequences K at a time, every remaining (sequence, seed) pair of a chunk in optimize_batch calls"""
    done = []
    K = args.batch_sequences
    for c0 in range(0, len(mine), K):
        chunk = mine[c0:c0 + K]
        todo = {}                                            # sequence -> seeds whose file is still missing
        for seq_name in chunk:
            for seed in seeds:
                out_file = out_file_of(args.out_dir, seq_name, seed)
                if args.cached and os.path.exists(out_file):
                    done.append((seq_name, seed, out_file, 0.0))
                else:
                    todo.setdefault(seq_name, []).append(seed)
        calls = []                                           # (sequences, seeds) of one optimize_batch call each
        if args.batch_seeds:
            by_seeds = {}
            for seq_name, ss in todo.items():
                by_seeds.setdefault(tuple(ss), []).append(seq_name)
            calls = [(seqs, list(ss)) for ss, seqs in by_seeds.items()]
        else:
            for seed in seeds:
                seqs = [q for q, ss in todo.items() if seed in ss]
                if seqs:
                    calls.append((seqs, [seed]))
        in_dicts = {}
        for seqs, ss in calls:
            for q in seqs:
                if q not in in_dicts:
                    in_dicts[q] = load(q)
            dicts = [in_dicts[q] for q in seqs]
            t0 = time.perf_counter()
            outs = model.optimize_batch(dicts, ss)           # sets the RNGs of every pair itself
            n = len(seqs) * len(ss)
            dt = (time.perf_counter() - t0) / n
            for seq_name, row in zip(seqs, outs):
                for seed, out_dict in zip(ss, row):
                    out_file = out_file_of(args.out_dir, seq_name, seed)
                    os.makedirs(os.path.dirname(out_file), exist_ok=True)
                    with open(out_file, 'wb') as f:
                        pickle.dump(out_dict, f)
                    done.append((seq_name, seed, out_file, dt))
                    if not args.quiet:
                        print(f'[rank {rank}] seed {seed} {seq_name}: {dt * 1e3:.1f} ms (batch of {n}) -> {out_file}', flush=True)
    return done


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--cfg', default='glamr_3dpw')
    ap.add_argument('--out_dir', default='out/3dpw')
    ap.add_argument('--seeds', default='1')
    ap.add_argument('--gpu', type=int, default=0)
    ap.add_argument('--cached', type=int, default=0)
    ap.add_argument('--pose_root', default='out/3dpw', help='<pose_root>/<seq>/pose_est/pose.pkl or <pose_root>/<seq>.pkl')
    ap.add_argument('--gt_pose_root', default=None)
    ap.add_argument('--sequences', default='', help='comma-separated sequence names (default: everything under pose_root)')
    ap.add_argument('--synthetic', type=int, default=0, help='generate this many seeded HybrIK-shaped sequences instead of reading pose.pkl')
    ap.add_argument('--frames', type=int, default=300)
    ap.add_argument('--persons', type=int, default=1)
    ap.add_argument('--gaps', action='store_true', help='synthetic sequences with occlusion gaps')
    ap.add_argument('--real_assets', action='store_true', help='with --synthetic: still load SMPL files / checkpoints from disk')
    ap.add_argument('--batch_seeds', action='store_true', help='optimise all seeds of a sequence in one optimize_seeds call')
    ap.add_argument('--batch_sequences', type=int, default=0,
                    help='optimise K sequences of this rank at a time in one optimize_batch call (0: one sequence at a time)')
    ap.add_argument('--quiet', action='store_true')
    return ap.parse_args(argv)


def main(argv=None):
    args = parse(argv)
    t0 = time.perf_counter()
    done = run(args)
    wall = time.perf_counter() - t0
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    busy = sum(d[3] for d in done)
    print(f'[rank {rank}/{world}] {len(done)} sequence runs, optimize() {busy:.3f} s, wall {wall:.3f} s', flush=True)


if __name__ == '__main__':
    main()
