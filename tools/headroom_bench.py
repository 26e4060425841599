"""Time the memory headroom written by the search kernels, and the two views built on it, on one GPU.

In one process, alternating:
  - api.cost_het_cluster on c3_homo64_mpl6 and c4_het128, with and without headroom=True (host clock around the call,
    which ends in a device synchronisation);
  - metis_headroom_select and metis_headroom_front alone on the same results (CUDA events around --launches launches);
  - HetSearchResult.breakdown(slice(None), per_stage=False), the replay that was the only source of every candidate's
    headroom before.
Prints one JSON line with the card's name, power limit and max SM clock beside the times (seconds; best of --reps after
one warm-up).  A device-listed 512-GPU space is not measured here.  Usage: python tools/headroom_bench.py [--reps 5]
"""
import argparse
import itertools
import json
import os
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

import numpy as np  # noqa: E402

from breakdown_bench import _card  # noqa: E402


def _call(name, root, headroom):
    from metis_b200 import api
    from metis_b200.arguments import parse_args
    from metis_b200.data_loader import ProfileDataLoader
    from metis_b200.gpu_cluster import GPUCluster
    from metis_b200.utils import ModelConfig
    from metis_b200.workloads import WORKLOADS, materialize, profile_file_order
    w = WORKLOADS[name]
    materialize(w, root)
    cluster = GPUCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
    profile, _ = ProfileDataLoader(os.path.join(root, 'profile'), profile_file_order(w)).load_profile_data_all()
    cfg = ModelConfig(model_name='t', num_layers=w.num_layers, sequence_length=w.sequence_length,
                      vocab_size=w.vocab_size, hidden_size=w.hidden_size, attention_head_size=32)
    args = parse_args(w.cli_args(root))
    volume = api.GPTActivationAndParam(cfg, profile['model']['parameters'])
    # bench.py's node sequences: the order of set(device types) (quirk Q4) would change the space from process to process
    seqs = list(itertools.permutations(w.device_types()))

    def run(with_headroom=headroom):
        return api.cost_het_cluster(args, cluster, profile, cfg, api.HeteroCostEstimator(profile, cfg, volume, cluster),
                                    api.LayerLoadBalancer(cluster, profile, cfg, args.gbs), node_sequences=seqs,
                                    device='cuda:0', headroom=with_headroom)
    return run


def _timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def _kernel_ms(launch, launches):
    import torch
    s = torch.cuda.current_stream()
    launch(s)
    s.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s)
    for _ in range(launches):
        launch(s)
    b.record(s)
    b.synchronize()
    return a.elapsed_time(b) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--launches', type=int, default=50)
    opt = ap.parse_args()
    import torch
    from metis_b200 import api
    out = dict(_card())
    for name in ('c3_homo64_mpl6', 'c4_het128'):
        run = _call(name, tempfile.mkdtemp(), False)
        run(False), run(True)                                 # warm-up of both paths
        plain, with_h, head_s = [], [], []
        for _ in range(opt.reps):                             # alternating
            t, _r = _timed(lambda: run(False))
            plain.append(t)
            t, res = _timed(lambda: run(True))
            with_h.append(t)
            head_s.append(res.timings['headroom_s'])
        res.ranked(1)
        idx = res._index()
        x = float(np.median(res.headroom))
        select_ms = _kernel_ms(lambda s: idx.launch_select(x, 100, s), opt.launches)
        front_ms = _kernel_ms(lambda s: idx.launch_front(s), opt.launches)
        bd = []
        for _ in range(opt.reps):
            t, _b = _timed(lambda: res.breakdown(slice(None), per_stage=False))
            bd.append(t)
        t_front, (pos, _c, _h) = _timed(res.pareto)
        t_sel, _sel = _timed(lambda: res.ranked(100, min_headroom=x))
        out[name] = dict(candidates=len(res), call_s=min(plain), call_headroom_s=min(with_h),
                         call_headroom_extra_pct=100.0 * (min(with_h) / min(plain) - 1.0),
                         headroom_copy_s=min(head_s), select_kernels_ms=select_ms, front_kernels_ms=front_ms,
                         front_len=len(pos), pareto_call_s=t_front, ranked100_min_headroom_call_s=t_sel,
                         breakdown_replay_s=min(bd), replay_over_kernels=min(bd) / (select_ms / 1e3 + front_ms / 1e3))
        api.release_engines()
        torch.cuda.empty_cache()
    out['device_listed_512'] = 'not measured'
    print(json.dumps(out))


if __name__ == '__main__':
    main()
