"""ase_b200 -- H100-native (sm_90a) engine for the PPO + adversarial update hot path of nv-tlabs/ASE.

The CUDA library (ase_b200/csrc/libase_b200.so, C ABI in include/ase_b200.h) is the product; this package
is the thin host-side mirror of the reference's agent / env helper interfaces.  Touching anything but
`ase_b200.build` without the built library raises: there is no CPU fallback."""
import importlib

_LAZY = {'lib': '.lib', 'ops': '.ops', 'learner': '.learner', 'agent': '.agent', 'synthetic_env': '.synthetic_env',
         'replay_buffer': '.replay_buffer', 'build': '.build', 'motion_lib': '.motion_lib', 'configs': '.configs',
         'dist_utils': '.dist_utils', 'player': '.player'}
__all__ = ['lib', 'ops', 'Learner', 'param_names', 'build']


def __getattr__(name):
    if name in _LAZY:
        return importlib.import_module(_LAZY[name], __name__)
    if name in ('Learner', 'param_names'):
        return getattr(importlib.import_module('.learner', __name__), name)
    raise AttributeError(name)
