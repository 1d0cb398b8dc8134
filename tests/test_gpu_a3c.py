"""GPU parity tests of the A3C learner: every call goes through the C-ABI (``drl_a3c_*``) and is compared with the
float64 oracle to 1e-4 relative by tests/a3c_parity.py; same ReLU-kink handling and Adam check as tests/apex_parity.py."""
import numpy as np
import pytest
import torch

from a3c_parity import compare_step
from oracle import a3c_torch as at
from parity import failures

pytestmark = pytest.mark.gpu


def _check(errs):
    bad = failures(errs)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1])[:10]


@pytest.mark.parametrize("mode", [1, 2])
def test_step_small(native, mode):
    _check(compare_step(3, A=4, math_mode=mode))


def test_step_reference_config(native):
    """config.json:2-41: one unroll of trajectory = 32 transitions, 4 actions."""
    _check(compare_step(32, A=4))


@pytest.mark.parametrize("B,A", [(1, 2), (7, 18)])
def test_step_ragged(native, B, A):
    _check(compare_step(B, A=A))


def test_three_steps_soft_asymmetric_cuda_graph(native):
    _check(compare_step(4, A=4, steps=3, reward_clipping="soft_asymmetric", use_cuda_graph=True))


def test_agent_train_and_act(native):
    from distributed_reinforcement_learning_b200.agent import a3c
    kw = dict(input_shape=[84, 84, 4], num_action=4, discount_factor=0.997, start_learning_rate=1e-4,
              end_learning_rate=0.0, learning_frame=1000000000, baseline_loss_coef=1.0, entropy_coef=0.05,
              gradient_clip_norm=40.0, reward_clipping="abs_one", model_name="learner", learner_name="learner")
    ag = a3c.Agent(**kw)
    ag.set_session(None)
    b = at.make_transitions(8, seed=3)
    L = at.Learner(at.unflatten_params(ag._params, torch.float32, num_action=4), torch.float64, num_action=4)
    for _ in range(2):
        got = ag.train(*[b[k] for k in at.TRAIN_FIELDS])
    ref = None
    res = L.train(*[b[k] for k in at.TRAIN_FIELDS])
    assert len(got) == 4 and all(np.isfinite(got))
    assert ag.num_env_frames == 2
    action, policy, max_prob = ag.get_policy_and_action(b["state"][0], 1)
    assert policy.shape == (4,) and abs(policy.sum() - 1) < 1e-5 and max_prob == policy[action]
    pol, val = ag._engine.act(b["state"][:3], b["previous_action"][:3])
    assert pol.shape == (3, 4) and val.shape == (3,)
