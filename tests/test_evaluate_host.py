"""Host side of evaluation (Trainer.evaluate): the argument rules of the episode quota (ic3_rollout_io.episodes) and of
greedy actions (ic3_policy_cfg.greedy) at the C ABI, the command-line flags, the evaluation line and the checkpoint's
'eval' key.  No GPU: every refused call returns before any device work."""
import ctypes

import numpy as np
import torch

E_RANGE, E_ARG = -2, -4
FAKE = 0x1000                      # never dereferenced: validation fails first


def pp_step(lib, _lib, **io):
    st = _lib.PPState(loc=FAKE, reached=FAKE, done=FAKE, success=FAKE, episode=FAKE, tick=FAKE)
    cfg = _lib.PPCfg(B=4, N=3, dim=5, vision=1, mode=0, naction=5, env_id0=0, enemy_comm=0, seed=1)
    r = _lib.RolloutIO(**dict(dict(t_ep=FAKE, fresh=FAKE, alive_next=FAKE, stat_episodes=FAKE, halted=FAKE, max_steps=20),
                              **io))
    return lib.ic3_pp_step(ctypes.byref(cfg), ctypes.byref(st), FAKE, 1, FAKE, None, FAKE, ctypes.byref(r), None)


def tj_step(lib, _lib, **io):
    st = _lib.TJState(loc=FAKE, alive=FAKE, wait=FAKE, route_id=FAKE, route_pos=FAKE, last_act=FAKE, completed=FAKE,
                      cars_in_sys=FAKE, has_failed=FAKE, tick=FAKE)
    cfg = _lib.TJCfg(B=4, N=5, vision=1, h=7, w=7, G=2, P=1, Lmax=7, outside_cls=4, car_cls=6, vocab=7, npath=2,
                     spawn_thr=1, env_id0=0, seed=1, grid=FAKE, route_len=FAKE, route_cells=FAKE, vocab_type=0)
    r = _lib.RolloutIO(**dict(dict(t_ep=FAKE, fresh=FAKE, alive_next=FAKE, stat_episodes=FAKE, halted=FAKE, max_steps=20),
                              **io))
    return lib.ic3_tj_step(ctypes.byref(cfg), ctypes.byref(st), FAKE, 1, None, FAKE, None, FAKE, ctypes.byref(r), None)


def test_episode_quota_rules(built_lib):
    from ic3net_b200 import _lib
    lib = _lib.load()
    for step in (pp_step, tj_step):
        assert step(lib, _lib, episodes=-1) == E_RANGE, step
        assert step(lib, _lib, episodes=2, batch_size=10) == E_ARG, step
        assert step(lib, _lib, episodes=2, halted=None) == E_ARG, step
        assert step(lib, _lib, episodes=2, stat_episodes=None) == E_ARG, step
    assert b"contradict" in lib.ic3_strerror(E_ARG)


def test_greedy_random_policy_is_refused(built_lib):
    from ic3net_b200 import _lib
    lib = _lib.load()
    hd = (ctypes.c_int32 * _lib.MAX_HEADS)(5, 2, 0, 0)
    cfg = _lib.PolicyCfg(B=4, N=3, nheads=2, head_dim=hd, greedy=1)
    io = _lib.PolicyIO(value=FAKE, logp=FAKE, action=FAKE)
    assert lib.ic3_random_policy_step(ctypes.byref(cfg), ctypes.byref(io), None, None) == E_ARG


def test_flags_parse():
    from ic3net_b200 import main as m
    p = m.build_parser()
    a = p.parse_args([])
    assert (a.eval_every, a.eval_episodes, a.eval_nenvs, a.eval_greedy) == (0, 1, None, False)
    a = p.parse_args(['--eval_every', '5', '--eval_episodes', '3', '--eval_nenvs', '256', '--eval_greedy'])
    assert (a.eval_every, a.eval_episodes, a.eval_nenvs, a.eval_greedy) == (5, 3, 256, True)


def test_eval_line_normalises_like_the_epoch_log():
    from ic3net_b200 import main as m
    stat = dict(num_episodes=10, num_steps=200, steps_taken=200, success=7, reward=np.array([1.0, 2.0]),
                comm_action=np.array([100.0, 50.0]))
    line = m.eval_line(stat, True, 2, 5)
    assert line.startswith('Eval (greedy, 2 episodes × 5 slots): ')
    assert 'Success 0.70' in line and 'Steps-taken 20.00' in line
    assert 'Reward [0.1 0.2]' in line and 'Comm-Action [0.5  0.25]' in line
    assert stat['success'] == 7                         # the raw sums are left as they are
    line = m.eval_line(dict(num_episodes=4, num_steps=8, steps_taken=8, reward=np.array([2.0])), False, 1, 4)
    assert line.startswith('Eval (sampled, 1 episodes') and 'Success' not in line


class _Opt(object):
    def __init__(self):
        self.state = {'steps': 3}

    def state_dict(self):
        return dict(self.state)

    def load_state_dict(self, s):
        self.state = dict(s)


def test_checkpoint_round_trips_with_and_without_eval(tmp_path):
    from ic3net_b200 import main as m
    net = torch.nn.Linear(3, 2)
    log = m.make_log()
    m.update_log(log, dict(num_episodes=2, num_steps=10, reward=np.array([1.0]), success=1, steps_taken=10))
    evals = [(1, dict(num_episodes=8, success=5, reward=np.array([0.5, 1.5])))]
    with_eval, without = str(tmp_path / 'a.pt'), str(tmp_path / 'b.pt')
    m.save_checkpoint(with_eval, net, log, _Opt(), evals)
    m.save_checkpoint(without, net, log, _Opt())
    with m._utils_alias():
        assert 'eval' not in torch.load(without, weights_only=False)
    for path, want in ((with_eval, evals), (without, [])):
        net2, log2, opt2 = torch.nn.Linear(3, 2), m.make_log(), _Opt()
        opt2.state = {}
        got = m.load_checkpoint(path, net2, log2, opt2)
        assert torch.equal(net2.weight, net.weight) and opt2.state == {'steps': 3}
        assert log2['success'].data == log['success'].data
        assert len(got) == len(want)
        for (e1, s1), (e2, s2) in zip(got, want):
            assert e1 == e2 and sorted(s1) == sorted(s2)
            for k in s1:
                assert np.array_equal(s1[k], s2[k])
