"""Host side of resuming a run (main.py --resumable / --resume): the checkpoint keeps the reference's keys, both files
of a save are replaced atomically, a sidecar is matched to its checkpoint, and the run fingerprint names what differs.
No GPU needed."""
import os

import pytest
import torch

from ic3net_b200 import main as m
from ic3net_b200.trainer import check_fingerprint


class _Net(object):
    def __init__(self, w):
        self.w = w

    def state_dict(self):
        return {'w': torch.full((3,), float(self.w))}


class _Opt(object):
    def __init__(self, steps):
        self.steps = steps

    def state_dict(self):
        st = {0: {'step': torch.tensor(float(self.steps)), 'square_avg': torch.ones(3)}} if self.steps else {}
        return {'state': st, 'param_groups': [dict(lr=1e-3, alpha=0.97, eps=1e-6, params=[0])]}


def _log(epochs):
    log = m.make_log()
    for _ in range(epochs):
        m.update_log(log, {'reward': 1.0, 'num_episodes': 1})
    return log


def _run(ep=1, update=0):
    return dict(ep=ep, update=update, stat=None, state=dict(fingerprint={'seed': 7}, ranks=[{'env': None}]))


def _load(path):
    with m._utils_alias():
        return torch.load(path, weights_only=False)


def test_plain_save_writes_the_reference_keys_and_no_sidecar(tmp_path):
    path = str(tmp_path / 'ck.pt')
    m.save_checkpoint(path, _Net(1), _log(1), _Opt(2))
    assert set(_load(path)) == {'policy_net', 'log', 'trainer'}
    assert sorted(os.listdir(str(tmp_path))) == ['ck.pt']        # no sidecar, no temporary left behind


def test_resumable_save_writes_a_matching_sidecar(tmp_path):
    path = str(tmp_path / 'ck.pt')
    m.save_checkpoint(path, _Net(1), _log(3), _Opt(6), run=_run(ep=3))
    assert set(_load(path)) == {'policy_net', 'log', 'trainer'}      # the checkpoint is what --load and the reference read
    run = m.read_run_file(path)
    assert (run['steps'], run['epochs'], run['ep'], run['update']) == (6, 3, 3, 0)
    assert run['version'] == m.RUN_FILE_VERSION and run['state']['fingerprint'] == {'seed': 7}
    assert m.checkpoint_position(_load(path)) == (6, 3)
    assert sorted(os.listdir(str(tmp_path))) == ['ck.pt', 'ck.pt.run']


def test_interrupted_save_leaves_the_previous_pair(tmp_path):
    path = str(tmp_path / 'ck.pt')
    m.save_checkpoint(path, _Net(1), _log(1), _Opt(2), run=_run(ep=1))
    before = [open(p, 'rb').read() for p in (path, path + '.run')]

    def fail(p):
        with open(p, 'wb') as f:
            f.write(b'partial')
        raise KeyboardInterrupt                 # a kill while the second file is being written
    with pytest.raises(KeyboardInterrupt):
        m.write_atomic([(path, lambda p: torch.save({'new': 1}, p)), (path + '.run', fail)])
    assert [open(p, 'rb').read() for p in (path, path + '.run')] == before
    # the same through save_checkpoint: a sidecar that cannot be written (an unpicklable stat) leaves both files alone
    bad = _run(ep=2)
    bad['stat'] = {'reward': lambda: 0}
    with pytest.raises(Exception):
        m.save_checkpoint(path, _Net(5), _log(2), _Opt(4), run=bad)
    assert [open(p, 'rb').read() for p in (path, path + '.run')] == before
    assert sorted(os.listdir(str(tmp_path))) == ['ck.pt', 'ck.pt.run']


def test_sidecar_of_another_checkpoint_is_refused(tmp_path):
    a, b = str(tmp_path / 'a.pt'), str(tmp_path / 'b.pt')
    m.save_checkpoint(a, _Net(1), _log(1), _Opt(2), run=_run(ep=1))
    m.save_checkpoint(b, _Net(2), _log(2), _Opt(4), run=_run(ep=2))
    os.replace(a + '.run', b + '.run')          # the new checkpoint beside the old sidecar
    with pytest.raises(ValueError, match=r'does not belong .* after 2 optimizer steps and 1 epochs, the checkpoint '
                                         r'after 4 and 2'):
        m.resume_checkpoint(b, m.read_run_file(b), None, m.make_log(), None)


def test_missing_sidecar_is_refused(tmp_path):
    path = str(tmp_path / 'ck.pt')
    m.save_checkpoint(path, _Net(1), _log(1), _Opt(2))
    with pytest.raises(FileNotFoundError, match=r'ck\.pt\.run .*--resumable'):
        m.read_run_file(path)


def test_fingerprint_comparison_names_every_differing_field():
    fp = dict(env_name='predator_prey', nenvs=64, world=1, seed=3, grad_impl='kernels')
    check_fingerprint(fp, dict(fp))
    with pytest.raises(ValueError) as e:
        check_fingerprint(fp, dict(fp, nenvs=128, seed=4, use_graph=True))
    msg = str(e.value)
    assert "nenvs (stored 64, now 128)" in msg and "seed (stored 3, now 4)" in msg
    assert "use_graph (stored None, now True)" in msg and "env_name" not in msg and "world" not in msg


@pytest.mark.parametrize('extra, message', [(['--resume', 'x.pt', '--load', 'x.pt'], 'takes no --load'),
                                            (['--resumable'], 'give --save')])
def test_cli_refuses_flag_combinations(capsys, extra, message):
    with pytest.raises(SystemExit):
        m.main(['--env_name', 'predator_prey', '--nagents', '3', '--dim', '5'] + extra)
    assert message in capsys.readouterr().err
