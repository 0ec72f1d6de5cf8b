"""bench.py contract pieces that run without a GPU: the reference arm (`--impl reference`) prints ONE JSON line with the
same metric / unit / higher_is_better / config keys as our arm plus impl, cpu_baseline and a zero-copy e2e object, and under
a multi-rank launch only rank 0 works."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(env_extra=None):
    env = dict(os.environ)
    env.update(env_extra or {})
    return subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--workload',
                           'h2o-ccpvdz-direct', '--steps', '1', '--warmup', '0'], capture_output=True, text=True, env=env,
                          timeout=300)


def test_reference_arm_json_line():
    p = _run()
    assert p.returncode == 0, p.stderr
    lines = [l for l in p.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d['impl'] == 'reference' and d['metric'] == 'J/K Fock-build wall-s/iter' and d['unit'] == 's'
    assert d['higher_is_better'] is False and d['vs_baseline'] is None and d['dtype'] == 'f64'
    assert d['config']['workload'] == 'h2o-ccpvdz-direct' and d['config']['nao'] == 24
    cb = d['cpu_baseline']
    assert cb['kind'] in ('reference', 'port') and cb['cores'] >= 1 and abs(cb['value'] - d['value']) < 1e-12
    assert d['e2e'] == {'value': d['value'], 'unit': 's', 'h2d_bytes_per_step': 0, 'd2h_bytes_per_step': 0}
    assert abs(d['ms_per_step'] - 1e3 * d['value']) < 1e-9


def test_reference_arm_other_ranks_idle():
    p = _run({'RANK': '1', 'WORLD_SIZE': '2', 'LOCAL_RANK': '1'})
    assert p.returncode == 0 and p.stdout.strip() == ''


def test_df_records_have_their_parity_fixtures():
    """Every DF configuration the bench appends to its line has its at-size oracle fixture committed."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    import bench
    import df_size_check as S
    for name, *_ in bench.DF_EXTRAS:
        fixtures = bench.SIZE_FIXTURE[name]
        for f in fixtures:
            if f is not None:
                z = S.load(f)
                assert z is not None, f
                assert int(z['nocc']) == bench.WORKLOADS[name]['nocc']


def test_dump_outputs(tmp_path):
    """--dump-outputs: float64 .npy per array, large arrays as the same seeded sample of 2^20 elements every time."""
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    small = np.arange(12.0).reshape(3, 4)
    big = np.random.RandomState(5).standard_normal(bench.DUMP_SAMPLE_BYTES // 8 + 1)
    for d in ('a', 'b'):
        bench.dump_outputs(str(tmp_path / d), 'w_', {'vj': small, 'vk': big})
    assert np.load(tmp_path / 'a' / 'w_vj.npy').dtype == np.float64
    assert (np.load(tmp_path / 'a' / 'w_vj.npy') == small).all()
    a, b = np.load(tmp_path / 'a' / 'w_vk.npy'), np.load(tmp_path / 'b' / 'w_vk.npy')
    assert a.shape == (1 << 20,) and (a == b).all() and np.isin(a, big).all()
