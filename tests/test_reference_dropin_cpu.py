"""Drop-in check against the reference's registry: `register_into_reference()` must make the registry the reference's
tools build from (`embodiedscan.registry.MODELS`) produce the esb200 classes from the reference's UNMODIFIED model configs.
The `model = dict(...)` of each config file is stored in tests/golden/reference_model_configs.json (Python literals,
written by `tests/golden/make_golden.py model_configs`); the registry is the mmengine stand-in of tests/golden/refstubs.py,
installed as `embodiedscan.registry` for the duration of the test. Like the reference, which registers its own classes
under these names first, the stand-in starts with a placeholder under every name; building one means
`register_into_reference()` did not override it."""
import ast
import json
import os
import sys
import types

import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CONFIGS = json.load(open(os.path.join(GOLD, 'reference_model_configs.json')))


def load_config(cfg_file):
    """The stored `model = dict(...)` of a reference config file."""
    return ast.literal_eval(CONFIGS[cfg_file])


@pytest.mark.parametrize('cfg_file,cls_name', [
    ('configs/detection/mv-det3d_8xb4_embodiedscan-3d-284class-9dof.py', 'SparseFeatureFusionSingleStage3DDetector'),
    ('configs/detection/cont-det3d_8xb1_embodiedscan-3d-284class-9dof.py', 'Embodied3DDetector'),
    ('configs/occupancy/mv-occ_8xb1_embodiedscan-occ-80class.py', 'DenseFusionOccPredictor'),
    ('configs/occupancy/cont-occ_8xb1_embodiedscan-occ-80class.py', 'EmbodiedOccPredictor'),
    ('configs/grounding/mv-grounding_8xb12_embodiedscan-vg-9dof.py', 'SparseFeatureFusion3DGrounder'),
    ('configs/grounding/mv-grounding_8xb12_embodiedscan-vg-9dof_fcaf-coder.py', 'SparseFeatureFusion3DGrounder'),
])
def test_reference_registry_builds_esb200_from_unmodified_configs(cfg_file, cls_name, monkeypatch):
    if GOLD not in sys.path:
        sys.path.insert(0, GOLD)
    import refstubs
    pkg = types.ModuleType('embodiedscan')
    reg = types.ModuleType('embodiedscan.registry')
    reg.MODELS, reg.TASK_UTILS = refstubs.Registry('model'), refstubs.Registry('task util')
    pkg.registry = reg
    monkeypatch.setitem(sys.modules, 'embodiedscan', pkg)
    monkeypatch.setitem(sys.modules, 'embodiedscan.registry', reg)

    import embodiedscan_b200
    from embodiedscan_b200.registry import MODELS, TASK_UTILS, register_into_reference

    def placeholder(name):
        def init(self, *args, **kwargs):
            raise AssertionError(f'the reference class {name} was built: register_into_reference() did not override it')
        return type(name, (), {'__init__': init})

    for ours, theirs in ((MODELS, reg.MODELS), (TASK_UTILS, reg.TASK_UTILS)):
        for name in ours._module_dict:
            theirs.register_module(name=name, module=placeholder(name))
    register_into_reference()
    model_cfg = load_config(cfg_file)
    assert model_cfg['type'] == cls_name
    for sub in ('backbone', 'neck'):                      # pretrained-checkpoint URLs need a network
        if isinstance(model_cfg.get(sub), dict):
            model_cfg[sub].pop('init_cfg', None)
    model = reg.MODELS.build(model_cfg)
    assert type(model).__module__.startswith('embodiedscan_b200'), type(model)
    assert type(model) is getattr(embodiedscan_b200, cls_name, None) or type(model).__name__ == cls_name
    names = dict(model.named_parameters())
    assert any(k.endswith('.kernel') for k in names) and 'backbone_3d.conv1.kernel' in names
