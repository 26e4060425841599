#!/usr/bin/env python3
"""Generate tests/golden/search_noise_<workload>.npz - the search what-if goldens - by executing the UNMODIFIED
reference (SamsungLabs/Metis @ ed41176) with make_golden.py's harness (its reference import and objects):

    METIS_REFERENCE=<checkout> PYTHONHASHSEED=0 python tests/golden/make_search_noise_golden.py [workload ...]

For each of make_noise_golden.py's SAMPLES samples P_j = metis_b200.search.noisy_profile(profile, SIGMA, SEED, j) of the
reference loader's profile, the reference's whole search (cost_het_cluster.py:21-50) under P_j: a HeteroCostEstimator
and a LayerLoadBalancer built from P_j (so its norm_layer_duration comes from P_j's first-listed entry, quirk Q3), the
workload's args, cluster and node sequences.  Recorded per sample:
  * status    '' or the type name of the exception that aborts the search; 'hang' for a sample the oracle says never
              terminates (load_balancer.py:96-104), which is screened first and not run in the reference (meta
              'oracle_derived' lists those samples)
  * count     len(estimate_costs)
  * best      the first entry of sorted(estimate_costs, key=cost): ordinal, step, ns_idx, device groups, dp, tp,
              batches, layer partition, num_repartition and the cost (its bits survive the float64 array)
  * kept      the searched best (the first entry of the workload golden's sorted candidates) held fixed under P_j:
              cost, headroom and exception codes from noise_<workload>.npz at that candidate's position
and each sample's sha256 (oracle_profile.sha256).  meta 'other_winner' lists the samples whose winner is not the
searched one.
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
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)

import make_golden as mg                                        # noqa: E402
import make_noise_golden as mn                                  # noqa: E402
import oracle_profile as op                                     # noqa: E402
from metis_b200.search import noisy_profile                    # noqa: E402
from metis_b200.workloads import WORKLOADS, materialize, profile_file_order  # noqa: E402
from oracle import metis_oracle as orc                         # noqa: E402

WORKLOADS_DONE = ['mix32', 'rough_q10']


def reference_search(ref, args, cluster, model_config, prof, seqs):
    """cost_het_cluster.py:21-50 of the reference under ``prof``: (rows in estimate_costs order, exception name or '')."""
    DeviceType = ref['utils'].DeviceType
    volume = ref['activation_parameter'].GPTActivationAndParam(model_config, prof['model']['parameters'])
    try:
        estimator = ref['cost_estimator'].HeteroCostEstimator(prof, model_config, volume, cluster)
        balancer = ref['load_balancer'].LayerLoadBalancer(cluster, prof, model_config, args.gbs)
    except Exception as exc:                                   # noqa: BLE001 - the caller's construction raises
        return [], type(exc).__name__
    gen = ref['plan'].InterStagePlanGenerator(device_types=set(cluster.get_device_types()),
                                              num_devices=cluster.get_total_num_devices(), gbs=args.gbs,
                                              num_layers=args.num_layers, variance=args.min_group_scale_variance,
                                              max_permute_len=args.max_permute_len)
    gen.node_sequences = [tuple(DeviceType[n] for n in seq) for seq in seqs]   # pin quirk Q4 to the golden's order
    rows = []
    with contextlib.redirect_stdout(io.StringIO()):
        for ordinal, inter in enumerate(gen):
            try:
                perf = ref['device_group'].StagePerformance(model_config, prof, cluster, inter)
                rank_map = perf.get_device_placement()
                intra_gen = ref['plan'].IntraStagePlanGenerator(inter, perf, balancer, args.max_profiled_tp_degree,
                                                                args.max_profiled_batch_size)
                step = 0
                while intra_gen.has_next:
                    intra = intra_gen.next()
                    try:
                        cost = estimator.get_cost(inter, intra.strategies, intra.layer_partition, rank_map)
                        rows.append((ordinal, step, inter.ns_idx, list(inter.device_groups), list(intra.strategies),
                                     inter.batches, list(intra.layer_partition), intra.num_repartition, cost))
                    except KeyError:                           # cost_het_cluster.py:47
                        pass
                    step += 1
            except Exception as exc:                           # noqa: BLE001 - aborts the reference search (Q8)
                return rows, type(exc).__name__
    return rows, ''


def golden_search_noise_workload(name: str):
    z = np.load(os.path.join(HERE, f'{name}.npz'))
    meta = json.loads(str(z['meta']))
    arr = {k: z[k] for k in z.files if k != 'meta'}
    nz = np.load(os.path.join(HERE, f'noise_{name}.npz'))
    nmeta = json.loads(str(nz['meta']))
    assert (nmeta['seed'], nmeta['sigma'], nmeta['samples']) == (mn.SEED, mn.SIGMA, mn.SAMPLES)
    searched = int(np.argsort(arr['cost'], kind='stable')[0])
    w = WORKLOADS[name]
    ref = mg.import_reference()
    with tempfile.TemporaryDirectory() as root:
        digest = materialize(w, root)
        assert digest == meta['inputs_sha256']
        args, cluster, base, _types, model_config, _volume = mg.build_objects(ref, w.cli_args(root),
                                                                              profile_file_order(w))
        seqs = meta['node_sequences']
        ocl = orc.OracleCluster(os.path.join(root, 'hostfile'), os.path.join(root, 'clusterfile.json'))
        K = mn.SAMPLES
        scen = [noisy_profile(base, mn.SIGMA, mn.SEED, j) for j in range(K)]
        status, count = [], np.zeros(K, dtype=np.int64)
        smax = int(arr['nstage'].max()) + 8
        best = dict(ordinal=np.full(K, -1, np.int64), step=np.zeros(K, np.int64), ns_idx=np.zeros(K, np.int64),
                    batches=np.zeros(K, np.int64), nrep=np.zeros(K, np.int64), cost=np.full(K, np.nan),
                    nstage=np.zeros(K, np.int64), groups=np.zeros((K, smax), np.int64),
                    dp=np.zeros((K, smax), np.int64), tp=np.zeros((K, smax), np.int64),
                    part=np.zeros((K, smax + 1), np.int64))
        derived, other = [], []
        for j, prof in enumerate(scen):
            model = orc.OracleModel(w.num_layers, w.hidden_size, w.sequence_length, w.vocab_size,
                                    prof['model']['parameters'])
            try:
                orc.het_search(prof, ocl, model, [tuple(s) for s in seqs], w.gbs, w.num_layers, w.variance,
                               w.max_permute_len, w.max_tp, w.max_bs)
            except RuntimeError:                               # the reference would not terminate: not run
                status.append('hang')
                derived.append(j)
                continue
            except Exception:                                  # noqa: BLE001 - the reference reports its own
                pass
            rows, exc = reference_search(ref, args, cluster, model_config, prof, seqs)
            status.append(exc)
            if exc:
                continue
            count[j] = len(rows)
            if not rows:
                continue
            r = sorted(rows, key=lambda kv: kv[-1])[0]          # cost_het_cluster.py:76, a stable sort
            S = len(r[3])
            best['ordinal'][j], best['step'][j], best['ns_idx'][j], best['batches'][j] = r[0], r[1], r[2], r[5]
            best['nrep'][j], best['cost'][j], best['nstage'][j] = r[7], r[8], S
            best['groups'][j, :S] = r[3]
            best['dp'][j, :S] = [d for d, _ in r[4]]
            best['tp'][j, :S] = [t for _, t in r[4]]
            best['part'][j, :S + 1] = r[6]
            if (r[0], r[1]) != (int(arr['ordinal'][searched]), int(arr['step'][searched])):
                other.append(j)
    out = dict(count=count, kept_cost=nz['costs'][:, searched], kept_headroom=nz['headroom'][:, searched],
               kept_cost_exc=nz['cost_exc'][:, searched], kept_memory_exc=nz['memory_exc'][:, searched],
               **{f'best_{k}': v for k, v in best.items()})
    m = {'workload': name, 'inputs_sha256': digest, 'seed': mn.SEED, 'sigma': mn.SIGMA, 'samples': K,
         'sample_sha256': [op.sha256(p) for p in scen], 'status': status, 'oracle_derived': derived,
         'searched': [int(arr['ordinal'][searched]), int(arr['step'][searched])], 'other_winner': other,
         'python': sys.version.split()[0]}
    mg.save(f'search_noise_{name}', m, out)
    print(f'search_noise_{name}: status {status}, counts {count.tolist()}, other winners {other}', file=sys.stderr)


def main():
    names = sys.argv[1:] or WORKLOADS_DONE
    sys.argv = sys.argv[:1]
    if os.environ.get('PYTHONHASHSEED') != '0':
        os.environ['PYTHONHASHSEED'] = '0'
        os.execv(sys.executable, [sys.executable, os.path.abspath(__file__)] + names)
    for name in names:
        golden_search_noise_workload(name)


if __name__ == '__main__':
    main()
