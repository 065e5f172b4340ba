"""CPU: host side of the 16-bit feature-map gathers -- the transfer plan of host-resident maps by element size, and
the refusal of map types the gathers do not read (engine and C ABI)."""
import types

import pytest

import gather_checks as GC

torch = pytest.importorskip("torch")


def _fp32_zero_copy_lines(s):
    """The line count of the in-place reader for 4-byte maps, as the plan has always computed it."""
    row = s.W * 4
    lines = min(s.k, -(-((s.k - 1) * row + s.k * 4) // 128) + 1) if s.k > 1 else 1
    return s.N * s.c * lines


def _maps(shapes, dtype):
    # meta tensors: numel() and element_size() without the memory
    return [dict(fmap_host=torch.empty((s.nbatch * s.B, s.c, s.H, s.W), dtype=dtype, device="meta")) for s in shapes]


def test_fp32_maps_keep_their_plan(monkeypatch):
    """4-byte maps: the same line counts and the same per-layer plan as a map described by numel() alone."""
    from cpb200 import pruner

    monkeypatch.delenv("CPB200_DMA_MAX_MB", raising=False)
    monkeypatch.delenv("CPB200_DMA_RATIO", raising=False)
    shapes = GC.all_shapes()
    for s in shapes:
        assert pruner.zero_copy_lines(s) == pruner.zero_copy_lines(s, 4) == _fp32_zero_copy_lines(s)

    class NumelOnly:
        def __init__(self, n):
            self._n = n

        def numel(self):
            return self._n

    plain = [dict(fmap_host=NumelOnly(s.nbatch * s.B * s.c * s.H * s.W)) for s in shapes]
    assert pruner.h2d_plan(shapes, _maps(shapes, torch.float32), True) == pruner.h2d_plan(shapes, plain, True)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_16bit_maps_halve_the_dma_and_count_their_own_lines(monkeypatch, dtype):
    import cpb200
    from cpb200 import pruner

    monkeypatch.delenv("CPB200_DMA_MAX_MB", raising=False)
    monkeypatch.delenv("CPB200_DMA_RATIO", raising=False)
    shapes = cpb200.synth.vgg16_layers()
    d32, d16 = _maps(shapes, torch.float32), _maps(shapes, dtype)
    for s, a, b in zip(shapes, d32, d16):
        assert b["fmap_host"].numel() * b["fmap_host"].element_size() * 2 == \
            a["fmap_host"].numel() * a["fmap_host"].element_size()
        assert pruner.zero_copy_lines(s, 2) <= pruner.zero_copy_lines(s, 4)
    by_name = {s.name: s for s in shapes}
    # conv4_2 (W = 28, k = 3): a window spans 2 * 28 * 4 + 12 = 236 bytes in fp32 (3 lines), 118 bytes in 16 bit (2)
    assert pruner.zero_copy_lines(by_name["conv4_2"], 4) == 5000 * 512 * 3
    assert pruner.zero_copy_lines(by_name["conv4_2"], 2) == 5000 * 512 * 2
    plan16 = pruner.h2d_plan(shapes, d16, True)
    for s, d, p in zip(shapes, d16, plan16):  # the plan's rule with the 16-bit bytes and lines
        nbytes = d["fmap_host"].numel() * 2
        dma = nbytes <= 300e6 and nbytes / 50e9 + 1e-4 < 0.8 * pruner.zero_copy_lines(s, 2) / pruner.ZC_LINES_PER_S
        assert p == ("dma" if dma else "zc"), s.name
    assert {s.name: p for s, p in zip(shapes, plan16)}["conv5_3"] == "dma"
    assert pruner.h2d_plan(shapes, d16, "zc") == ["zc"] * len(shapes)
    assert pruner.h2d_plan(shapes, d16, "copy") == ["dma"] * len(shapes)


@pytest.mark.parametrize("dtype", [torch.float64, torch.int32, torch.uint8])
def test_engine_refuses_maps_the_gathers_cannot_read(dtype):
    from cpb200 import engine

    assert [engine.fmap_dtype_code(t) for t in (torch.float32, torch.bfloat16, torch.float16)] == [0, 2, 3]
    with pytest.raises(TypeError):
        engine.fmap_dtype_code(dtype)
    fm = torch.zeros(2, 4, 5, 5, dtype=dtype)
    r = torch.zeros(1, 2, dtype=torch.int32)
    stub = types.SimpleNamespace()  # the type check comes before any device work
    with pytest.raises(TypeError):
        engine.Engine.patch_gather(stub, fm, r, r, 2, 2, 3, 1, 1)
    with pytest.raises(TypeError):
        engine.Engine.point_gather(stub, fm, r, r, 2, 2)


def test_c_abi_rejects_bad_fmap_dtype_before_touching_the_device():
    """cp_*_gather_typed check the dtype code first: CP_F64 and unknown codes return CP_ERR_INVALID with a message;
    the three map types pass that check (and here fail on the NULL handle instead)."""
    import cpb200

    ffi, lib = cpb200._cabi.load()
    assert (lib.CP_F32, lib.CP_F64, lib.CP_BF16, lib.CP_F16) == (0, 1, 2, 3)
    NULL = ffi.NULL

    def patch(dt):
        return lib.cp_patch_gather_typed(NULL, NULL, dt, 1, 1, 4, 5, 5, 0, NULL, NULL, 1, 3, 1, 1, 1, NULL, 36, NULL)

    def point(dt):
        return lib.cp_point_gather_typed(NULL, NULL, dt, 1, 1, 4, 5, 5, 0, NULL, NULL, 1, NULL, 4, NULL)

    for call in (patch, point):
        for dt in (lib.CP_F64, 7, -1):
            assert call(dt) == lib.CP_ERR_INVALID
            assert b"dtype" in ffi.string(lib.cp_last_error())
        for dt in (lib.CP_F32, lib.CP_BF16, lib.CP_F16):
            assert call(dt) == lib.CP_ERR_INVALID
            assert b"NULL argument" in ffi.string(lib.cp_last_error())
