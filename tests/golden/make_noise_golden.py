#!/usr/bin/env python3
"""Generate tests/golden/noise_<workload>.npz - the profile-noise what-if goldens - by executing the UNMODIFIED
reference (SamsungLabs/Metis @ ed41176) at fixed arguments, with make_golden.py's harness (its reference import and
objects), in the pattern of make_profile_golden.py:

    METIS_REFERENCE=<checkout> PYTHONHASHSEED=0 python tests/golden/make_noise_golden.py [workload ...]

For every candidate of the workload's search golden (tests/golden/<workload>.npz) and each of SAMPLES samples
metis_b200.search.noisy_profile(profile, SIGMA, SEED, j) of the reference loader's profile:
  * cost      HeteroCostEstimator(P_j, model_config, GPTActivationAndParam(model_config, P_j['model']['parameters']),
              cluster).get_cost(plan, strategies, layer_partition, rank_device_map), NaN when it raises
  * headroom  min(LayerLoadBalancer(cluster, P_j, model_config, gbs)._detect_out_of_memory(
              _get_stage_memory_demand(layer_partition, strategies, device_groups,
              _device_types_by_node_sequence(node_sequence), gbs, batches),
              StagePerformance(...).get_device_group_memory_capacity())[1]), NaN when the demand raises
  * the type of each exception (oracle_profile.EXC) and the sha256 of every sample (oracle_profile.sha256), so that
    the tests can rebuild the same dicts from the seed and check that they did.
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(REPO, 'tests'))
sys.path.insert(0, HERE)

import make_golden as mg                                        # noqa: E402
import oracle_profile as op                                     # noqa: E402
from metis_b200.search import noisy_profile                    # noqa: E402
from metis_b200.workloads import WORKLOADS, materialize, profile_file_order  # noqa: E402

WORKLOADS_DONE = ['mix32', 'rough_q10']
SEED = 0x5eed_0f_9e01_5e
SAMPLES = 8
# every field noisy, fb_sync by device type; memory wide enough that some samples make some candidates stop fitting
SIGMA = {'layer-computes': 0.2, 'memory': 0.3, 'fb_sync': {'A100': 0.1, 'H100': 0.25, 'V100': 0.05, 'T4': 0.3}}


def golden_noise_workload(name: str):
    z = np.load(os.path.join(HERE, f'{name}.npz'))
    meta = json.loads(str(z['meta']))
    arr = {k: z[k] for k in z.files if k != 'meta'}
    w = WORKLOADS[name]
    ref = mg.import_reference()
    DeviceType = ref['utils'].DeviceType
    with tempfile.TemporaryDirectory() as root:
        digest = materialize(w, root)
        assert digest == meta['inputs_sha256']
        order = profile_file_order(w)
        args, cluster, base, _types, model_config, _volume = mg.build_objects(ref, w.cli_args(root), order)
        seqs = meta['node_sequences']
        scen = [noisy_profile(base, SIGMA, SEED, j) for j in range(SAMPLES)]
        cands = op.candidate_args(arr, seqs)
        K, n = len(scen), len(cands)
        costs, head = np.full((K, n), np.nan), np.full((K, n), np.nan)
        cexc, mexc = np.zeros((K, n), dtype=np.int8), np.zeros((K, n), dtype=np.int8)
        names = {}
        with contextlib.redirect_stdout(io.StringIO()):
            for j, prof in enumerate(scen):
                volume = ref['activation_parameter'].GPTActivationAndParam(model_config, prof['model']['parameters'])
                est = ref['cost_estimator'].HeteroCostEstimator(prof, model_config, volume, cluster)
                llb = ref['load_balancer'].LayerLoadBalancer(cluster, prof, model_config, args.gbs)
                for i, (plan, strategies, part) in enumerate(cands):
                    inter = ref['plan'].InterStagePlan(ns_idx=int(arr['ns_idx'][i]),
                                                       node_sequence=[DeviceType[t] for t in plan['node_sequence']],
                                                       dg_idx=0, device_groups=plan['device_groups'],
                                                       num_stage=plan['num_stage'], batches=plan['batches'],
                                                       gbs=args.gbs)
                    perf = ref['device_group'].StagePerformance(model_config, prof, cluster, inter)
                    try:
                        costs[j, i] = est.get_cost(inter, strategies, part, perf.get_device_placement())
                    except Exception as e:                     # noqa: BLE001
                        cexc[j, i] = op.exc_code(e)
                        names[type(e).__name__] = names.get(type(e).__name__, 0) + 1
                    capa = perf.get_device_group_memory_capacity()
                    try:
                        types = llb._device_types_by_node_sequence(inter.node_sequence)
                        demand = llb._get_stage_memory_demand(part, strategies, inter.device_groups, types, args.gbs,
                                                              inter.batches)
                        head[j, i] = min(llb._detect_out_of_memory(demand, capa)[1])
                    except Exception as e:                     # noqa: BLE001
                        mexc[j, i] = op.exc_code(e)
    out = dict(costs=costs, headroom=head, cost_exc=cexc, memory_exc=mexc)
    m = {'workload': name, 'inputs_sha256': digest, 'seed': SEED, 'sigma': SIGMA, 'samples': SAMPLES,
         'sample_sha256': [op.sha256(p) for p in scen], 'cost_exceptions': names,
         'python': sys.version.split()[0]}
    mg.save(f'noise_{name}', m, out)
    print(f'noise_{name}: {n} candidates x {K} samples, usable per sample '
          f'{[int(((cexc[j] == 0) & (mexc[j] == 0) & (head[j] >= 0)).sum()) for j in range(K)]}, '
          f'get_cost exceptions {names}', file=sys.stderr)


def main():
    names = sys.argv[1:] or WORKLOADS_DONE
    sys.argv = sys.argv[:1]
    if os.environ.get('PYTHONHASHSEED') != '0':
        os.environ['PYTHONHASHSEED'] = '0'
        os.execv(sys.executable, [sys.executable, os.path.abspath(__file__)] + names)
    for name in names:
        golden_noise_workload(name)


if __name__ == '__main__':
    main()
