"""hold_b200.dropin adaptors carry the reference's own call signatures (SURVEY §8b).  Where $HOLD_REFERENCE names a checkout
of the reference they are compared with `inspect.signature` of the reference's classes, imported behind the harness
shims in a separate interpreter (the shims patch torch.Tensor.cuda); elsewhere only the committed copy of those signatures
(tests/golden/reference_signatures.json, written by this test when the reference is present) is checked."""
import inspect
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "reference_signatures.json")

PAIRS = {   # reference callable -> adaptor
    "src.engine.ray_sampler:ErrorBoundSampler.__init__": "hold_b200.dropin:ErrorBoundSampler.__init__",
    "src.engine.ray_sampler:ErrorBoundSampler.get_z_vals": "hold_b200.dropin:ErrorBoundSampler.get_z_vals",
    "src.engine.ray_sampler:UniformSampler.inverse_sample": "hold_b200.dropin:UniformInverseSphereSampler.inverse_sample",
    "src.model.mano.deformer:MANODeformer.forward": "hold_b200.dropin:MANODeformer.forward",
    "src.model.mano.deformer:MANODeformer.forward_skinning": "hold_b200.dropin:MANODeformer.forward_skinning",
    "src.model.obj.deformer:ObjectDeformer.forward": "hold_b200.dropin:ObjectDeformer.forward",
    "src.model.obj.deformer:ObjectDeformer.forward_skinning": "hold_b200.dropin:ObjectDeformer.forward_skinning",
    "src.networks.shape_net:ImplicitNet.forward": "hold_b200.model:ImplicitNet.forward",
    "src.networks.texture_net:RenderingNet.forward": "hold_b200.dropin:RenderingNetAdaptor.forward",
    "src.engine.volsdf_utils:sdf_func_with_deformer": "hold_b200.dropin:sdf_func_with_deformer",
}
CTORS = {   # constructors: the reference's positional parameters, then keyword-only extras for what the reference reads from disk
    "src.model.renderables.mano_node:MANONode.__init__": "hold_b200.dropin:MANONode.__new__",
    "src.model.renderables.object_node:ObjectNode.__init__": "hold_b200.dropin:ObjectNode.__new__",
    "src.model.renderables.background:Background.__init__": "hold_b200.dropin:Background.__new__",
    "src.hold.hold_net:HOLDNet.__init__": "hold_b200.dropin:HOLDNet.__new__",
}

_DUMP = r"""
import sys, json, inspect, importlib
sys.path.insert(0, %r); sys.path.insert(0, %r)
from oracle import ref_harness
ref_harness.install_shims()
sys.path.insert(0, ref_harness.REF + '/code'); sys.path.insert(0, ref_harness.REF)
out = {}
import types
class _Stub(types.ModuleType):          # third-party packages the reference imports but this container lacks (matplotlib, trimesh, ...)
    def __getattr__(self, k):
        if k.startswith('__'):
            raise AttributeError(k)
        return _Stub(self.__name__ + '.' + k) if k[0].islower() else type(k, (), {})
    def __call__(self, *a, **kw):
        return None
for _n in ('trimesh', 'cv2'):
    if _n in sys.modules and not hasattr(sys.modules[_n], '__file__'):
        sys.modules[_n] = _Stub(_n)
def _import(mod):
    for _ in range(40):
        try:
            return importlib.import_module(mod)
        except ModuleNotFoundError as e:
            name = e.name
            parts = name.split('.')
            for i in range(1, len(parts) + 1):
                sys.modules.setdefault('.'.join(parts[:i]), _Stub('.'.join(parts[:i])))
        except ImportError as e:       # `from pkg import compiled_extension` that is not built in the tree (src.libmise.mise)
            if getattr(e, 'name_from', None) is None or e.name not in sys.modules:
                raise
            setattr(sys.modules[e.name], e.name_from, _Stub(e.name + '.' + e.name_from))
            for k in [k for k in sys.modules if k.startswith('src.') and getattr(sys.modules[k], '__spec__', None) is not None and getattr(sys.modules[k].__spec__, '_initializing', False)]:
                del sys.modules[k]
    raise RuntimeError('cannot import ' + mod)
for spec in %r:
    mod, path = spec.split(':')
    obj = _import(mod)
    for part in path.split('.'):
        obj = getattr(obj, part)
    out[spec] = [[p.name, None if p.default is inspect._empty else repr(p.default)] for p in inspect.signature(obj).parameters.values()]
print('SIGS=' + json.dumps(out))
"""


def _sig(spec):
    import importlib

    mod, path = spec.split(":")
    obj = importlib.import_module(mod)
    for part in path.split("."):
        obj = getattr(obj, part)
    return [[p.name, None if p.default is inspect._empty else repr(p.default)] for p in inspect.signature(obj).parameters.values()]


def _reference_signatures():
    if os.path.isdir(os.environ.get("HOLD_REFERENCE", "")):
        r = subprocess.run([sys.executable, "-c", _DUMP % (ROOT, os.path.join(ROOT, "oracle"), list(PAIRS) + list(CTORS))], capture_output=True, text=True,
                           timeout=300, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-3000:]
        sigs = json.loads([l for l in r.stdout.splitlines() if l.startswith("SIGS=")][-1][5:])
        with open(GOLD, "w") as f:
            json.dump(sigs, f, indent=1, sort_keys=True)
        return sigs
    if not os.path.exists(GOLD):
        pytest.skip("no reference tree and no committed signature file")
    return json.load(open(GOLD))


def test_adaptors_have_the_reference_signatures():
    ref = _reference_signatures()
    for rspec, aspec in PAIRS.items():
        theirs, ours = ref[rspec], _sig(aspec)
        assert [p[0] for p in ours] == [p[0] for p in theirs], f"{aspec}: parameters {[p[0] for p in ours]} vs reference {[p[0] for p in theirs]}"
        assert [p[1] for p in ours] == [p[1] for p in theirs], f"{aspec}: defaults {[p[1] for p in ours]} vs reference {[p[1] for p in theirs]}"


def test_constructors_take_the_reference_arguments():
    """MANONode / ObjectNode / Background / HOLDNet: same positional parameters as the reference's __init__ (names and order);
    everything the adaptor adds is keyword-only."""
    ref = _reference_signatures()
    for rspec, aspec in CTORS.items():
        import importlib

        mod, path = aspec.split(":")
        obj = importlib.import_module(mod)
        for part in path.split("."):
            obj = getattr(obj, part)
        params = list(inspect.signature(obj).parameters.values())[1:]     # drop cls
        pos = [p.name for p in params if p.kind == p.POSITIONAL_OR_KEYWORD]
        extra = [p for p in params if p.kind != p.POSITIONAL_OR_KEYWORD]
        assert pos == [p[0] for p in ref[rspec]][1:], f"{aspec}: {pos} vs reference {[p[0] for p in ref[rspec]][1:]}"
        assert all(p.kind == p.KEYWORD_ONLY for p in extra), aspec


def test_constructor_rejects_another_architecture():
    from hold_b200 import dropin

    opt = {"implicit_network": dict(dropin._SUPPORTED["implicit_network"], multires=8), "rendering_network": dict(dropin._SUPPORTED["rendering_network"], d_in=14)}
    with pytest.raises(ValueError, match="multires"):
        dropin.MANONode({"n_images": 2}, opt, None, 3.0, "right", mano={})
