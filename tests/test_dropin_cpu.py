"""Drop-in proof for INTEGRATION.md section 2 (CPU only): a full-object checkpoint written by the REAL reference
(``torch.save({'model': model})``, train.py:424-435; stored as tests/golden/dropin_ckpt.pt.gz by oracle/gen_golden_dropin.py)
is unpickled into the shadow modules (``sys.modules['models.common'] = icafusion_b200.common`` etc.), goes through what
``attempt_load`` does (models/experimental.py:113-121: ``ckpt['model'].float().fuse().eval()``), a state_dict of the
reference's layout (tests/golden/dropin_reference.json) loads with ``strict=True`` and the unpickled model walks the product
path (dry run: meta tensors, every kernel launch planned, none issued)."""
import json
import os
import subprocess
import sys
import textwrap

from conftest import GOLDEN, ROOT


def _meta():
    with open(os.path.join(GOLDEN, "dropin_reference.json")) as f:
        return json.load(f)


def test_reference_checkpoint_unpickles_into_shadow_modules():
    meta = _meta()
    assert meta["model_module"] == "models.yolo_test"
    ckpt, mpath = os.path.join(GOLDEN, "dropin_ckpt.pt.gz"), os.path.join(GOLDEN, "dropin_reference.json")
    code = textwrap.dedent(f"""
        import gzip, io, json, sys, torch
        sys.path.insert(0, {ROOT!r})
        import icafusion_b200.common as C, icafusion_b200.yolo_test as Y
        from oracle.gen_golden_dropin import dropin_value
        import types
        pkg = types.ModuleType("models"); pkg.__path__ = []
        sys.modules["models"] = pkg                    # INTEGRATION.md section 2: shadow before anything imports the reference
        sys.modules["models.common"] = C
        sys.modules["models.yolo_test"] = Y
        from icafusion_b200 import ops
        meta = json.load(open({mpath!r}))
        ck = torch.load(io.BytesIO(gzip.decompress(open({ckpt!r}, "rb").read())), map_location="cpu", weights_only=False)
        m = ck["model"]
        assert type(m) is Y.Model and type(m.model[0]) is C.Conv and type(m.model[-1]) is Y.Detect, type(m)
        assert type(m.model[20]) is C.TransformerFusionBlock and type(m.model[20].crosstransformer[0].crossatt) is C.CrossAttention
        # the reference's state_dict layout, with the stored values: every tensor arrived where the reference put it
        want = {{}}
        got = m.state_dict()
        assert sorted(got) == [k for k, _, _ in meta["state_dict"]]
        for i, (k, shape, dtype) in enumerate(meta["state_dict"]):
            assert list(got[k].shape) == shape, k
            if got[k].is_floating_point():
                want[k] = torch.full(shape, dropin_value(i, k), dtype=torch.float16).float()
                assert torch.equal(got[k].float(), want[k]), k
            else:
                want[k] = got[k].clone()
        m = m.float().fuse().eval()                    # models/experimental.py:118
        assert not hasattr(m.model[0], "bn") and m.model[0].conv.bias is not None
        # a state_dict of the reference's (unfused) layout loads strictly into a freshly built shadow model
        fresh = Y.Model("yolov5s_Transfusion_kaist")
        missing = fresh.load_state_dict(want, strict=True)
        assert not missing.missing_keys and not missing.unexpected_keys
        fresh = fresh.eval().fuse()
        for (ka, va), (kb, vb) in zip(sorted(m.state_dict().items()), sorted(fresh.state_dict().items())):
            assert ka == kb and va.shape == vb.shape and torch.allclose(va.float(), vb.float(), atol=2e-3, rtol=2e-3), ka
        # the unpickled object drives the product path: dry-run walk (nothing launched), every conv plan accepted
        from icafusion_b200 import _lib
        import ctypes
        img = torch.empty(1, 3, 512, 640, dtype=torch.uint8, device="meta")
        with torch.no_grad(), ops.dry_run() as dr:
            z, logits, xs = m.half()(img, img)
        assert tuple(z.shape) == (1, 20160, 6) and len(xs) == 3
        convs = [w for n, a, w in dr.records if n == "icaf_conv2d_fwd"]
        assert len(convs) >= 60
        for w in convs:
            pl = _lib.ConvPlan()
            assert _lib.lib().icaf_conv2d_plan(ctypes.byref(w["geom"]), w["n_io"], 132, -1, ctypes.byref(pl)) == 0
        print("ok", len(dr.records))
    """)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, (out.stdout[-1000:], out.stderr[-3000:])
    assert out.stdout.strip().startswith("ok")


def test_shadow_modules_export_the_reference_names():
    """Every class the Transfusion YAMLs / pickles name exists in the shadow modules with the reference's constructor
    signature (parameter names and defaults, as recorded from the reference in tests/golden/dropin_reference.json)."""
    import inspect
    import icafusion_b200.common as C
    import icafusion_b200.yolo_test as Y
    meta = _meta()
    assert len(meta["common_classes"]) == 11
    for name in meta["common_classes"]:
        assert hasattr(C, name), name
    assert len(meta["signatures"]) == 9
    for name, want in meta["signatures"].items():
        b = inspect.signature(getattr(C, name).__init__)
        assert [[p.name, repr(p.default)] for p in b.parameters.values()] == want, name
    for name in ("Model", "Detect"):
        assert hasattr(Y, name)
    assert [p.name for p in inspect.signature(Y.Detect.__init__).parameters.values()] == meta["detect_params"]
