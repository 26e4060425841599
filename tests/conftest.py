import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, 'golden')
if REPO not in sys.path:
    sys.path.insert(0, REPO)


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (run on an H100 with -m gpu)')
    config.addinivalue_line('markers', 'slow: long-running CPU test')


def load_golden(name):
    """Returns (meta dict, arrays dict) of tests/golden/<name>.npz (made by make_golden.py)."""
    path = os.path.join(GOLDEN, f'{name}.npz')
    if not os.path.exists(path):
        pytest.skip(f'golden {name}.npz not generated')
    z = np.load(path, allow_pickle=False)
    meta = json.loads(str(z['meta']))
    return meta, {k: z[k] for k in z.files if k != 'meta'}


def golden_rows(arrays):
    """Unpack golden arrays into tuples comparable with oracle / product candidates."""
    out = []
    for i in range(len(arrays['cost'])):
        s = int(arrays['nstage'][i])
        out.append((int(arrays['ordinal'][i]), int(arrays['step'][i]), int(arrays['ns_idx'][i]),
                    [int(x) for x in arrays['groups'][i, :s]],
                    [(int(d), int(t)) for d, t in zip(arrays['dp'][i, :s], arrays['tp'][i, :s])],
                    int(arrays['batches'][i]),
                    [int(x) for x in arrays['part'][i, :s + 1]],
                    int(arrays['nrep'][i]), float(arrays['cost'][i])))
    return out


@pytest.fixture(scope='session')
def workload_dir(tmp_path_factory):
    """Materialise a named synthetic workload once per session; returns (Workload, root)."""
    from metis_b200.workloads import WORKLOADS, materialize
    cache = {}

    def get(name):
        if name not in cache:
            root = str(tmp_path_factory.mktemp(name))
            digest = materialize(WORKLOADS[name], root)
            cache[name] = (WORKLOADS[name], root, digest)
        return cache[name]
    return get


C1_DIR = os.path.join(GOLDEN, 'fixtures', 'c1')
