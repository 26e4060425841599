"""Time the two ways of listing a plan space's compositions and planning its windows, and their host memory.

  host    flatten.build_device_plan_space (metis_enum_compositions: every record on the host) + flatten.plan_windows
  device  metis_b200.listing.DeviceListing (the GPU lists them) + flatten.plan_listed_windows + the exact size of
          every window (one metis_list_window sizing pass each)

Each (mode, space) runs in a subprocess of its own so that its host peak RSS is its own.  Same budget and cost model as
a windowed search on an 80 GB card: 60 GB, (56.5, 1.25, 20.0) bytes per plan / row byte / record.  Prints one JSON
line per run; ``--out`` also writes them as a JSON list.

    python tools/listing_bench.py [--points 256:4,512:4,512:6] [--modes host,device] [--out FILE]
"""
import argparse
import json
import os
import resource
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL, BUDGET, LAYERS = (56.5, 1.25, 20.0), 60e9, 96


def run_one(mode: str, gpus: int, mpl: int) -> dict:
    sys.path.insert(0, REPO)
    from metis_b200 import flatten
    cap = min(gpus, LAYERS)
    out = {'mode': mode, 'gpus': gpus, 'variance': 0, 'mpl': mpl}
    if mode == 'host':
        t0 = time.perf_counter()
        space = flatten.build_device_plan_space(1, gpus, gpus, LAYERS, 0, mpl)
        t1 = time.perf_counter()
        windows = flatten.plan_windows(space, BUDGET, *MODEL)
        t2 = time.perf_counter()
        out.update(records=len(space.comp_recs))
    else:
        import torch
        from metis_b200 import listing
        torch.zeros(1, device='cuda:0')                       # CUDA context outside the timed region
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lst = listing.DeviceListing(gpus, cap, 0, mpl, 'cuda:0', max_ranges=cap + 1)
        t1 = time.perf_counter()
        space = flatten.listed_plan_space(1, gpus, gpus, LAYERS, lst.rows_per_stage)
        windows = flatten.plan_listed_windows(space, BUDGET, *MODEL, listing=lst)
        for w in windows:
            w.sized()
        t2 = time.perf_counter()
        out.update(records=sum(w.num_recs for w in windows), compositions=int(lst.comps_per_stage.sum()),
                   gpu=torch.cuda.get_device_name(0))
    out.update(plans=int(space.num_plans), rows_bytes=int(space.rows_total_bytes), windows=len(windows),
               listing_s=t1 - t0, planning_s=t2 - t1, host_peak_rss_bytes=resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024)
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--points', default='256:4,512:4,512:6', help='GPUS:MPL, comma-separated (1 type, variance 0)')
    ap.add_argument('--modes', default='host,device')
    ap.add_argument('--out')
    ap.add_argument('--one', help=argparse.SUPPRESS)          # MODE:GPUS:MPL, run in this process
    a = ap.parse_args()
    if a.one:
        mode, gpus, mpl = a.one.split(':')
        print(json.dumps(run_one(mode, int(gpus), int(mpl))))
        return
    results = []
    for point in a.points.split(','):
        gpus, mpl = point.split(':')
        for mode in a.modes.split(','):
            proc = subprocess.run([sys.executable, os.path.abspath(__file__), '--one', f'{mode}:{gpus}:{mpl}'],
                                  capture_output=True, text=True)
            line = proc.stdout.strip().splitlines()[-1] if proc.returncode == 0 and proc.stdout.strip() else None
            res = json.loads(line) if line else {'mode': mode, 'gpus': int(gpus), 'mpl': int(mpl),
                                                 'error': proc.stderr.strip().splitlines()[-1:]}
            print(json.dumps(res), flush=True)
            results.append(res)
    if a.out:
        with open(a.out, 'w') as fh:
            json.dump(results, fh, indent=1)


if __name__ == '__main__':
    main()
