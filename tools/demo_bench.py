"""Wall time of ``python -m sparsefusion_b200.demo`` from process start to exit, on synthetic inputs (``synthetic.write_demo_inputs``:
12-view toy scenes, random-weight checkpoints of the released configuration): model load, cache build, ``--max-itr`` iterations (the
last ``max_itr - 1001`` of them with the SDS target), scores and pictures, for 1 and for S scenes in one run.  Prints the card's name and
power limit with the times.

    python tools/demo_bench.py --max-itr 1100 --scenes 1 4
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--max-itr', type=int, default=1100)
    ap.add_argument('--scenes', type=int, nargs='+', default=[1, 4])
    a = ap.parse_args()
    from sparsefusion_b200.synthetic import write_demo_inputs
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True,
                          text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as d:
        p = write_demo_inputs(d, 'hydrant', n_scenes=max(a.scenes))
        for s in a.scenes:
            cwd = os.path.join(d, f'run{s}')
            os.makedirs(cwd)
            cmd = [sys.executable, '-m', 'sparsefusion_b200.demo', '-c', 'hydrant', '-r', p['root'], '-e', p['eft'], '-l', p['vldm'],
                   '-a', p['vae'], '--lpips', p['lpips'], '-i', ','.join(str(i) for i in range(s)), '--max-itr', str(a.max_itr)]
            t0 = time.perf_counter()
            out = subprocess.run(cmd, cwd=cwd, capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT))
            dt = time.perf_counter() - t0
            if out.returncode != 0:
                sys.stderr.write(out.stdout[-4000:] + out.stderr[-4000:])
                raise SystemExit(f'demo failed for {s} scenes')
            print(json.dumps(dict(scenes=s, max_itr=a.max_itr, seconds=round(dt, 1), card=card)), flush=True)


if __name__ == '__main__':
    main()
