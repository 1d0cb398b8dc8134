"""H100-native stand-in for the reference's ``model/actor_critic.py`` (the A3C network): parameter inventory of scope
'a3c' in TF layouts / TF variable order -- conv2d x3, dense x2 (action embedding), dense x3 (actor 3392 -> 256 -> 256 -> A,
softmax), dense x3 (critic 3392 -> 256 -> 256 -> 1).  The same body as ``model/apex_value.py`` with the two streams named
actor / critic; the graph (``network`` :28-39, ``build_network`` :41-56) is evaluated by ``drl_a3c_*`` through
``agent/a3c.py``."""
import numpy as np

from . import apex_value


def param_specs(num_action=4, input_shape=(84, 84, 4)):
    out = []
    for name, shape in apex_value.param_specs(num_action=num_action, input_shape=input_shape):
        name = name.replace("value", "actor").replace("mean", "critic")
        out.append((name, shape))
    return out


def param_count(**kw):
    return sum(int(np.prod(s)) for _, s in param_specs(**kw))


def init_params(seed=None, **kw):
    return apex_value.init_params(seed, **kw)
