"""Scripted opponents (reference: python/magent/builtin/rule_model/).

``RandomActor`` keeps the reference's semantics: uniform actions drawn from numpy's global generator on the host.
``RushActor`` and ``FleeActor`` are the engine's built-in scripted policies (include/magent_b200_ext.h
magent_b200_rule_actions), decided on the device.  They are not the reference's RushPredator / RunawayPrey, whose
decisions depend on glibc random() and read the observation in ways this package does not reproduce (DESIGN.md §9).
"""
import numpy as np


class RandomActor:
    """uniform random actions over the whole action space, drawn on the host"""

    def __init__(self, env, handle, *args, **kwargs):
        self.env = env
        self.handle = handle
        self.n_action = env.get_action_space(handle)[0]

    def infer_action(self, obs, *args, **kwargs):
        num = len(obs[0])
        return np.random.randint(self.n_action, size=num, dtype=np.int32)


class _RuleActor:
    policy = None

    def __init__(self, env, handle, target, seed=0):
        self.env = env
        self.handle = handle
        self.target = target
        self.seed = int(seed)

    def infer_action(self, obs=None, *args, **kwargs):
        """int32 (n,) in the order of set_action: the device's choice on the state as it is now; `obs` is not read"""
        return self.env.get_rule_actions(self.handle, self.target, self.policy, self.seed).copy()


class RushActor(_RuleActor):
    """attack the weakest target in reach, else step towards the nearest visible target, else a random legal action"""
    policy = "rush"


class FleeActor(_RuleActor):
    """step away from the nearest visible target, else a random legal action"""
    policy = "flee"
