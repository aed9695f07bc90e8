"""Host logic of bench.py's CPU legs (the reference arm measured beside the GPU arm)."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
  sys.path.insert(0, REPO)


def test_oracle_pool_two_processes():
  """Ray-sharded multi-process layout: two workers render their shards between a barrier and
  the last finish; the pool survives a second command and shuts down cleanly."""
  import bench
  pool = bench.OraclePool(2, 1, 'quarterhd-train', 128)
  try:
    assert pool.ok
    t1 = pool.run(64)
    t2 = pool.run(64)
    assert t1 and t1 > 0 and t2 and t2 > 0
  finally:
    pool.close()
  assert all(not p.is_alive() for p in pool.ps)


def test_reference_line_keys(monkeypatch, capsys):
  """--impl reference prints one JSON line with the contract's keys (tiny sample)."""
  import json
  import bench

  class FakeLayout:
    def __init__(self, wl_name, max_rays):
      pass

    def sample(self, budget_s):
      return (1000.0, 4, 256, 0.1, '256 rays, one process x 4 torch threads')

    def close(self):
      pass
  monkeypatch.setattr(bench, 'CpuLayout', FakeLayout)
  monkeypatch.setattr(sys, 'argv', ['bench.py', '--impl', 'reference', '--steps', '2', '--warmup', '1'])
  monkeypatch.setenv('RANK', '0')
  args = bench.parse_args()
  bench.run_reference(args)
  line = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  for k in ('impl', 'metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better',
            'config', 'cpu_baseline', 'e2e'):
    assert k in line
  assert line['impl'] == 'reference' and line['e2e']['h2d_bytes_per_step'] == 0
  assert line['cpu_baseline']['cores'] == 4 and line['value'] == 1000.0
