"""CPU: the uint8 stem ABI without a device (struct size, argument checks), the uint8 input helpers
of dataflow.py, and the reach of the GPU test's shape tables (stem_u8_cases.py)."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import stem_u8_cases as uc
import tail_cases as tc

_BASE = 1 << 20
_STEP = 0x100000
_ODD = 8          # 8 bytes past a 16-byte boundary
_IMAGENET = uc.NORMS["imagenet"]


def _u8(nat, Cout=32, mean=_IMAGENET[0], std=_IMAGENET[1], **conv):
    a = nat.StemConvU8()
    c = a.ev.conv
    c.N, c.H, c.W, c.Cout = 2, 36, 44, Cout
    c.x, c.w, c.y, c.dh, c.dw = (_BASE + i * _STEP for i in range(5))
    a.ev.scale, a.ev.shift, a.ev.act = _BASE + 5 * _STEP, _BASE + 6 * _STEP, 1
    for k, v in conv.items():
        setattr(c, k, v)
    a.mean[:] = mean
    a.std[:] = std
    return a


_INF, _NAN = float("inf"), float("nan")
_NORM_BAD = [dict(std=(0.229, 0.0, 0.225)), dict(std=(_NAN, 0.224, 0.225)),
             dict(std=(0.229, 0.224, _INF)), dict(std=(0.229, 0.224, -_INF)),
             dict(mean=(0.485, _NAN, 0.406)), dict(mean=(_INF, 0.456, 0.406))]
_FWD_BAD = [dict(Cout=12), dict(Cout=72), dict(Cout=0), dict(x=None), dict(N=0),
            dict(y=_BASE + 2 * _STEP + _ODD), dict(y=None), dict(w=None)] + _NORM_BAD
_WGRAD_BAD = [dict(Cout=12), dict(Cout=72), dict(Cout=24), dict(Cout=56), dict(x=None),
              dict(dh=_BASE + 3 * _STEP + _ODD), dict(dh=None), dict(dw=None)] + _NORM_BAD
_ENTRIES = [("yamb_stem_conv_u8_fwd", b) for b in _FWD_BAD] + \
    [("yamb_stem_conv_u8_eval_fwd", b) for b in _FWD_BAD] + \
    [("yamb_stem_conv_u8_wgrad", b) for b in _WGRAD_BAD]


def _refused(lib, rc):
    assert rc == -1, (rc, lib.yamb_last_error())
    assert lib.yamb_last_error() not in (b"", b"no CUDA device")


def test_struct_size(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    assert built_lib.yamb_struct_size(28) == C.sizeof(nat.StemConvU8) == 104
    assert C.sizeof(nat.StemConvU8) == C.sizeof(nat.StemConvEval) + 24


@pytest.mark.parametrize("fn,bad", _ENTRIES, ids=["%s-%d" % (f[10:], i) for i, (f, _) in
                                                   enumerate(_ENTRIES)])
def test_u8_refuses(built_lib, fn, bad):
    from yet_another_mobilenet_series_b200 import native as nat
    _refused(built_lib, getattr(built_lib, fn)(C.byref(_u8(nat, **bad)), None))


def test_u8_eval_refuses_act_and_coefficients(built_lib):
    from yet_another_mobilenet_series_b200 import native as nat
    for k, v in (("act", 5), ("act", -1), ("scale", None), ("shift", None)):
        a = _u8(nat)
        setattr(a.ev, k, v)
        _refused(built_lib, built_lib.yamb_stem_conv_u8_eval_fwd(C.byref(a), None))
    for fn in ("yamb_stem_conv_u8_fwd", "yamb_stem_conv_u8_wgrad", "yamb_stem_conv_u8_eval_fwd"):
        _refused(built_lib, getattr(built_lib, fn)(None, None))


def test_u8_well_formed_reaches_device_check(built_lib):
    """Unmodified arguments pass every check: without a device they get YAMB_ENODEV, so each
    refusal above is the check it names."""
    if built_lib.yamb_max_ctas() > 0:
        pytest.skip("a CUDA device is visible")
    from yet_another_mobilenet_series_b200 import native as nat
    for fn in ("yamb_stem_conv_u8_fwd", "yamb_stem_conv_u8_wgrad", "yamb_stem_conv_u8_eval_fwd"):
        for norm in uc.NORMS.values():
            rc = getattr(built_lib, fn)(C.byref(_u8(nat, mean=norm[0], std=norm[1])), None)
            assert rc == -2, (fn, rc, built_lib.yamb_last_error())
    rc = built_lib.yamb_stem_conv_u8_fwd(C.byref(_u8(nat, Cout=56, W=45)), None)
    assert rc == -2, built_lib.yamb_last_error()


# ---- dataflow --------------------------------------------------------------------------------------
def _images(n, H, W, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(n)]


@pytest.mark.parametrize("H,W", [(224, 224), (7, 5), (1, 3)])
def test_fast_collate_arrays(H, W):
    from yet_another_mobilenet_series_b200.dataflow import fast_collate
    imgs = _images(5, H, W)
    x, t = fast_collate([(a, i * 3) for i, a in enumerate(imgs)])
    assert x.shape == (5, 3, H, W) and x.dtype == torch.uint8
    assert x.stride() == (H * W * 3, 1, W * 3, 3)
    assert x.is_contiguous(memory_format=torch.channels_last)
    assert t.dtype == torch.int64 and t.tolist() == [0, 3, 6, 9, 12]
    want = np.stack(imgs)                                     # [N, H, W, 3]
    assert np.array_equal(x.permute(0, 2, 3, 1).numpy(), want)


def test_fast_collate_pil():
    Image = pytest.importorskip("PIL.Image")
    from yet_another_mobilenet_series_b200.dataflow import fast_collate
    imgs = _images(3, 9, 12, seed=1)
    x, t = fast_collate([(Image.fromarray(a), 1) for a in imgs])
    assert np.array_equal(x.permute(0, 2, 3, 1).numpy(), np.stack(imgs))
    assert x.is_contiguous(memory_format=torch.channels_last) and t.tolist() == [1, 1, 1]


def test_fast_collate_rejects_mixed_shapes():
    from yet_another_mobilenet_series_b200.dataflow import fast_collate
    with pytest.raises(ValueError):
        fast_collate([(np.zeros((4, 4, 3), np.uint8), 0), (np.zeros((4, 5, 3), np.uint8), 0)])
    with pytest.raises(ValueError):
        fast_collate([(np.zeros((4, 4), np.uint8), 0)])


def test_set_input_norm_is_a_plain_attribute():
    from yet_another_mobilenet_series_b200 import dataflow
    m = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3), torch.nn.BatchNorm2d(8))
    keys = list(m.state_dict().keys())
    dataflow.set_input_norm(m, *_IMAGENET)
    assert list(m.state_dict().keys()) == keys
    assert dataflow.input_norm_of(m) == _IMAGENET
    assert dataflow.input_norm_of(copy.deepcopy(m)) == _IMAGENET
    assert dataflow.input_norm_of(torch.nn.Linear(2, 2)) is None
    for mean, std in (((0.5, 0.5), (0.5, 0.5, 0.5)), ((0.5,) * 3, (0.5, 0.0, 0.5)),
                      ((float("nan"), 0.5, 0.5), (0.5,) * 3)):
        with pytest.raises(ValueError):
            dataflow.set_input_norm(m, mean, std)


@pytest.mark.parametrize("norm", sorted(uc.NORMS))
def test_host_normalize_is_torchvision(norm):
    """The twin the GPU test feeds the bf16 kernels is torchvision's ToTensor + Normalize, bf16."""
    tvf = pytest.importorskip("torchvision.transforms.functional")
    Image = pytest.importorskip("PIL.Image")
    u = np.concatenate([np.arange(256, dtype=np.uint8).reshape(16, 16)[..., None]] * 3, axis=2)
    u[..., 1] = u[..., 1][::-1]
    mean, std = uc.NORMS[norm]
    tv = tvf.normalize(tvf.to_tensor(Image.fromarray(u)), mean, std).to(torch.bfloat16)
    ours = uc.host_normalize(torch.from_numpy(u), uc.NORMS[norm]).permute(2, 0, 1)
    assert torch.equal(tv.view(torch.int16), ours.contiguous().view(torch.int16))


# ---- reach of the GPU tables -----------------------------------------------------------------------
def test_gpu_tables_reach_every_path():
    plans = [(c, tc.stem_plan(c.N, c.H, c.W)) for c in uc.DIRECT_CASES + uc.WALK_CASES]
    aligned = [c for c, _ in plans if uc.u8_aligned(c.W)]
    generic = [c for c, _ in plans if not uc.u8_aligned(c.W)]
    assert aligned and generic
    assert any((3 * c.W) % 2 for c in generic)                 # odd 3W
    assert any((3 * c.W) % 2 == 0 for c in generic)            # even 3W, not 4-byte rows
    for path in (aligned, generic):
        cut = [c for c in path if tc.stem_cut_edges(tc.stem_plan(c.N, c.H, c.W))]
        assert cut, path
        assert any(tc.stem_plan(c.N, c.H, c.W).tiles_w > 1 for c in path)
        walks = [c for c in path if c in uc.WALK_CASES]
        assert {c.Cout for c in walks} == set(tc.STEM_WGRAD_COUT), path
        for c in walks:
            p = tc.stem_plan(c.N, c.H, c.W)
            assert tc.stem_is_walk(p) and tc.stem_cut_edges(p), c
    for co in tc.STEM_FWD_COUT:
        assert any(c.Cout == co and uc.u8_aligned(c.W) for c in uc.DIRECT_CASES), co
    assert any(uc.u8_aligned(W) for _, _, W in uc.EVAL_SHAPES)
    assert any(not uc.u8_aligned(W) for _, _, W in uc.EVAL_SHAPES)
