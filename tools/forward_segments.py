#!/usr/bin/env python3
"""Developer tool: model a segmented prediction walk for the chain kernel's forward pass on every balancer run the
chain kernel makes, on the host (no GPU needed).

  python tools/forward_segments.py [workload ...] [--place demand]

Compiles tools/forward_segments.cpp with g++ into tools/_build/ (in the instantiation the GPU would pick for the
workload), runs the search's schedule over the whole plan space and prints, for G = 2, 4, 8 lane groups, three guesses
of a group's first start and overlaps K = 2, 4, 8: the window-miss rate at 32/G entries, how often a group's path meets
the true one at its boundary, later or never, and the modeled walk steps per run (the longest group's steps plus the
continuation after boundaries whose paths did not meet) against today's S - 1.  --place demand puts every window
around the end that the stage's demand predicts instead of the previous stage's length."""
import argparse
import ctypes
import itertools
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from metis_b200 import api, native  # noqa: E402
from metis_b200.arguments import parse_args  # noqa: E402
from metis_b200.data_loader import ProfileDataLoader  # noqa: E402
from metis_b200.gpu_cluster import GPUCluster  # noqa: E402
from metis_b200.utils import ModelConfig  # noqa: E402
from metis_b200.workloads import WORKLOADS, materialize, profile_file_order  # noqa: E402

SRC = os.path.join(ROOT, 'tools', 'forward_segments.cpp')
BUILD = os.path.join(ROOT, 'tools', '_build')


def tool(tier):
    out = os.path.join(BUILD, f'forward_segments_s{tier[0]}_l{tier[1]}_one{int(tier[2])}.so')
    os.makedirs(BUILD, exist_ok=True)
    subprocess.check_call(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared',
                           f'-DFS_MAXS={tier[0]}', f'-DFS_MAXL={tier[1]}', f'-DFS_ONE={int(tier[2])}', '-o', out, SRC])
    return ctypes.CDLL(out)


def run(name, place):
    w = WORKLOADS[name]
    tmp = tempfile.TemporaryDirectory()
    materialize(w, tmp.name)
    args = parse_args(w.cli_args(tmp.name))
    cluster = GPUCluster(args.hostfile_path, args.clusterfile_path)
    profile, _ = ProfileDataLoader(args.profile_data_path, profile_file_order(w)).load_profile_data_all()
    cfg = ModelConfig(model_name=args.model_name, num_layers=args.num_layers, sequence_length=args.sequence_length,
                      vocab_size=args.vocab_size, hidden_size=args.hidden_size,
                      attention_head_size=args.attention_head_size)
    balancer = api.LayerLoadBalancer(cluster, profile, cfg, args.gbs)
    seqs = list(itertools.permutations(w.device_types()))
    native.load_library()
    problem, space, _ = api.het_problem(args, cluster, profile, cfg, balancer, seqs)
    max_stage = int(space.blocks['num_stage'].max())
    one = len(w.device_types()) == 1
    # the instantiation metis_het_search picks (tests/hostsim_util.gpu_tier)
    tier = (64, 128, one) if max_stage <= 64 and w.num_layers <= 128 else \
        (96, 128, one) if max_stage <= 96 and w.num_layers <= 128 else (128, 256, one)
    lib = tool(tier)
    keep = dict(problem.arrays)
    keep.update(blocks=space.blocks, batches=space.batches, rows=space.rows)
    p = problem.as_struct(lambda n: keep[n].ctypes.data)
    s = space.as_struct(lambda n: keep[n].ctypes.data)
    print(f'{name}: {space.num_plans} plans, instantiation {tier}, window placement {place}', flush=True)
    rc = lib.forward_segments(ctypes.byref(p), ctypes.byref(s), ctypes.c_int(int(place == 'demand')))
    assert rc == 0, rc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('workloads', nargs='*', default=['c3_homo64_mpl6', 'c4_het128'])
    ap.add_argument('--place', choices=['span', 'demand'], default='span')
    ns = ap.parse_args()
    for name in ns.workloads:
        run(name, ns.place)


if __name__ == '__main__':
    main()
