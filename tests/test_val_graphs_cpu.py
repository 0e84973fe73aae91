"""In-place refresh of the packed-filter caches (engine.refresh_packed_) and the model / device checks of test.test(graphs=),
without a GPU: the dry-run forward packs every cache on the CPU."""
import copy

import pytest
import torch

from helpers import load_synth
from icafusion_b200.engine import refresh_packed_


def _packed_model(cfg="yolov5s_Transfusion_kaist", fuse=False):
    from icafusion_b200 import Model, ops
    m = Model(cfg).eval()
    load_synth(m, 3)
    if fuse:
        m.fuse()
    img = torch.empty(1, 3, 512, 640, dtype=torch.uint8, device="meta")
    with torch.no_grad(), ops.dry_run():
        m(img, img)
    return m


def _cached(model) -> dict:
    """Every tensor of every packed-filter cache, by (module name, cache, path)."""
    from icafusion_b200.ops import PackedConv
    out = {}

    def walk(where, v):
        if isinstance(v, PackedConv):
            for f in ("w", "bias", "colsum"):
                walk(where + (f,), getattr(v, f))
        elif isinstance(v, dict):
            for k in sorted(v, key=str):
                walk(where + (k,), v[k])
        elif isinstance(v, (tuple, list)):
            for i, x in enumerate(v):
                walk(where + (i,), x)
        elif torch.is_tensor(v):
            out[where] = v
    for name, m in model.named_modules():
        for cache in ("_icaf_pack", "_icaf_pack12"):
            c = m.__dict__.get(cache)
            if c is None:
                continue
            if cache == "_icaf_pack12":
                walk((name, cache), c[2])
            elif isinstance(c, dict):                       # Detect: level -> (key, pack)
                walk((name, cache), {i: e[1] for i, e in c.items()})
            else:
                walk((name, cache), c[1])
    return out


def _fresh(model) -> dict:
    """The caches a model with these exact parameters and buffers packs from scratch."""
    from icafusion_b200 import ops
    src = {id(m): {k: m.__dict__.pop(k) for k in [k for k in m.__dict__ if k.startswith("_icaf_")]} for m in model.modules()}
    try:
        twin = copy.deepcopy(model)
    finally:
        for m in model.modules():
            m.__dict__.update(src[id(m)])
    img = torch.empty(1, 3, 512, 640, dtype=torch.uint8, device="meta")
    with torch.no_grad(), ops.dry_run():
        twin(img, img)
    return _cached(twin)


@pytest.mark.parametrize("fuse", [False, True], ids=["bn", "fused"])
def test_refresh_keeps_addresses_and_equals_a_fresh_pack(fuse):
    from icafusion_b200.common import C3, Conv, CrossAttention, CrossTransformerBlock, TransformerFusionBlock
    m = _packed_model(fuse=fuse)
    before = _cached(m)
    kinds = {type(mod) for mod in m.modules() if "_icaf_pack" in mod.__dict__ or "_icaf_pack12" in mod.__dict__}
    assert {Conv, C3, CrossAttention, CrossTransformerBlock, TransformerFusionBlock} <= kinds
    assert any(k[1] == "_icaf_pack12" for k in before) and any(k[-1] == "colsum" for k in before)
    ptrs = {k: t.data_ptr() for k, t in before.items()}
    values = {k: t.clone() for k, t in before.items()}
    assert refresh_packed_(m) == 0                              # nothing moved: nothing re-packed
    g = torch.Generator().manual_seed(7)
    with torch.no_grad():                                        # what ModelEMA.update does: every floating entry moves
        for v in m.state_dict().values():
            if v.dtype.is_floating_point and v.numel():
                v.mul_(0.75).add_(torch.rand(v.shape, generator=g) * 0.01)
    n = refresh_packed_(m)
    after = _cached(m)
    assert after.keys() == before.keys() and n > len(before) // 8
    moved = [k for k, t in after.items() if t.data_ptr() != ptrs[k] or t is not before[k]]
    assert not moved, moved[:5]
    fresh = _fresh(m)
    assert fresh.keys() == after.keys()
    for k, t in after.items():
        assert torch.equal(t, fresh[k]), k
    assert sum(not torch.equal(t, values[k]) for k, t in after.items()) > len(after) // 2
    assert refresh_packed_(m) == 0


def test_refresh_follows_a_batchnorm_buffer_alone():
    m = _packed_model()
    conv = m.model[1]
    w = conv.__dict__["_icaf_pack"][1].w
    old = w.clone()
    with torch.no_grad():
        conv.bn.running_var.mul_(4.0)
    assert refresh_packed_(m) == 1
    assert conv.__dict__["_icaf_pack"][1].w is w and not torch.equal(w, old)
    assert torch.equal(w, _fresh(m)[("model.1", "_icaf_pack", "w")])


def test_refresh_refuses_a_new_shape():
    m = _packed_model()
    det = m.model[-1]
    old = det.m[0]
    det.m[0] = torch.nn.Conv2d(old.in_channels, old.out_channels + 32, 1)
    with pytest.raises(ValueError, match="does not fit the cached"):
        refresh_packed_(m)
    m = _packed_model()
    conv = m.model[1]
    conv.conv.stride = (1, 1)
    with torch.no_grad():
        conv.bn.bias.add_(1.0)
    with pytest.raises(ValueError, match="stride changed"):
        refresh_packed_(m)


def test_decode_values_follow_detect_anchors():
    from icafusion_b200.engine import decode_values
    m = _packed_model()
    det = m.model[-1]
    a, strides = decode_values(m)
    assert a == det.__dict__["_icaf_anchor_px"][1] and strides == [8.0, 16.0, 32.0]
    with torch.no_grad():
        det.anchor_grid.mul_(2.0)
    assert decode_values(m) == ([[2 * x for x in lv] for lv in a], strides)


def test_copy_packed_refuses_what_would_rebind():
    from icafusion_b200 import ops
    a = ops.pack_conv_weight(torch.ones(32, 8, 3, 3), torch.zeros(32), 1, 1, ops.ACT_SILU)
    same = ops.pack_conv_weight(torch.full((32, 8, 3, 3), 2.0), torch.ones(32), 1, 1, ops.ACT_SILU)
    w = a.w
    assert ops.copy_packed_(a, same) is a and a.w is w and torch.equal(a.w, same.w)
    for bad in (ops.pack_conv_weight(torch.ones(32, 8, 3, 3), torch.zeros(32), 2, 1, ops.ACT_SILU),     # stride
                ops.pack_conv_weight(torch.ones(32, 8, 3, 3), None, 1, 1, ops.ACT_SILU),               # no bias
                ops.pack_conv_weight(torch.ones(64, 8, 3, 3), torch.zeros(64), 1, 1, ops.ACT_SILU)):   # shape
        with pytest.raises(ValueError):
            ops.copy_packed_(a, bad)
    with pytest.raises(ValueError):
        ops.copy_packed_({"a": torch.zeros(2)}, {"b": torch.zeros(2)})
    with pytest.raises(ValueError):
        ops.copy_packed_(torch.zeros(4, dtype=torch.float16), torch.zeros(4))


def test_test_refuses_graphs_of_another_model_or_device(tmp_path):
    from icafusion_b200 import Model, ops
    from icafusion_b200 import test as T
    from icafusion_b200.engine import ValidationGraphs
    data = {"nc": 1, "names": ["person"]}
    with ops.dry_run():
        a = Model("yolov5n_Transfusion_kaist").to("meta").eval()
        b = Model("yolov5n_Transfusion_kaist").to("meta").eval()
        g = ValidationGraphs(a)
        with pytest.raises(ValueError, match="another model"):
            T.test(data, model=b, dataloader=[], save_dir=tmp_path, graphs=g)
    a.to_empty(device="cpu")
    with pytest.raises(ValueError, match="now on cpu"):
        T.test(data, model=a, dataloader=[], save_dir=tmp_path, graphs=g)
    with pytest.raises(RuntimeError, match="CUDA"):
        ValidationGraphs(b.to_empty(device="cpu"))
    with pytest.raises(ValueError, match="eval"):
        ValidationGraphs(Model("yolov5n_Transfusion_kaist").train())
    with pytest.raises(TypeError):
        ValidationGraphs(torch.nn.Linear(2, 2))
