"""Expected output digest of bench.py's input batch 0 (tests/golden/bench_digest.json).

Runs the ORACLE with the product's bf16 rounding points (oracle.recognize(policy='bf16')) in the build container on exactly
the weights (bench.build_model(), seed 1234) and inputs (bench.synthetic_batch(32, 0)) of the benchmark and stores the sha1 of
the int64 1-best ids [32, 1, 60].  bench.py hashes the ids the CUDA path produced for the same batch and reports
`validation.match`; tests/test_gpu_bench_config.py asserts the id equality itself on 4 utterances.

    python tools/make_bench_digest.py          # ~2 min of CPU
"""
import hashlib
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from oracle import beam_search as obs  # noqa: E402

torch.set_num_threads(min(8, os.cpu_count() or 1))
model = bench.build_model()
sd, params = bench.flat_state_dict(model), bench.model_params()
x, mask = bench.synthetic_batch(bench.B_PER_GPU, 0)
ids = []
with torch.no_grad():
    for b0 in range(0, bench.B_PER_GPU, 4):
        nb, _, _, _ = obs.recognize(x[b0:b0 + 4], mask[b0:b0 + 4], sd, params, beam=bench.BEAM, nbest=1, max_len=bench.MAX_LEN,
                                    penalty=bench.PENALTY, lamda=bench.LAMDA, policy='bf16')
        ids.append(nb)
        print('utterances', b0, '..', b0 + 3, 'distinct tokens in 1-best', [len(set(r.tolist())) for r in nb[:, 0]], flush=True)
ids = torch.cat(ids, 0).to(torch.int64).contiguous()
path = os.path.join(ROOT, 'tests', 'golden', 'bench_digest.json')
try:
    out = json.load(open(path))
except Exception:
    out = {}
out.update({'oracle_sha1': hashlib.sha1(ids.numpy().tobytes()).hexdigest(), 'shape': list(ids.shape),
            'generator': 'tools/make_bench_digest.py (oracle, policy bf16); gpu_* keys: validation.ids_sha1 of bench.py on an H100',
            'oracle_ids': ids[:, 0].tolist()})
with open(path, 'w') as f:
    json.dump(out, f)
print({k: v for k, v in out.items() if k != 'oracle_ids'})
