"""CPU checks of the GEMM dispatcher through otb_gemm_config (host only, no GPU): which N tile width otb_linear launches
and which epilogue / output combinations it refuses.  Only facts that hold whatever the SM count are checked here; the
GPU file tests/test_gpu_gemm.py runs every configuration the dispatcher can answer."""
import pytest

EPIS = range(9)   # OTB_EPI_BIAS .. OTB_EPI_TANH
MS = (1, 64, 129, 512, 513, 7968)
NS = (8, 64, 100, 256, 384, 768, 4234)


@pytest.fixture(scope='module')
def ops():
    from opentransformer_b200 import build
    build.build()
    from opentransformer_b200 import ops
    yield ops
    ops.set_tile_policy('latency')


@pytest.fixture(params=['latency', 'throughput'])
def policy(request, ops):
    ops.set_tile_policy(request.param)
    yield request.param
    ops.set_tile_policy('latency')


def test_glu_always_takes_128(ops, policy):
    for M in MS:
        for N in NS:
            for f32 in (False, True):
                assert ops.gemm_config(M, N, ops.EPI_GLU, f32) == 128, (M, N, f32)


def test_residual_layernorm_tile_is_the_row(ops, policy):
    for M in MS:
        for N in (64, 128, 256):
            assert ops.gemm_config(M, N, ops.EPI_RESID_LN) == N
        for N in (8, 32, 100, 192, 384, 512):
            with pytest.raises(RuntimeError, match=r'otb_gemm_config.*N in \{64,128,256\}'):
                ops.gemm_config(M, N, ops.EPI_RESID_LN)


def test_residual_epilogues_refuse_fp32_output(ops, policy):
    with pytest.raises(RuntimeError, match='fused residual\\+LayerNorm epilogue writes bf16'):
        ops.gemm_config(300, 256, ops.EPI_RESID_LN, True)
    for M, N in ((1, 64), (300, 256), (7968, 384)):
        with pytest.raises(RuntimeError, match='residual epilogue writes bf16'):
            ops.gemm_config(M, N, ops.EPI_RESID, True)
        assert ops.gemm_config(M, N, ops.EPI_RESID, False) in (64, 128)


def test_every_answer_is_a_compiled_tile(ops, policy):
    for epi in EPIS:
        for f32 in (False, True):
            for M in MS:
                for N in NS:
                    try:
                        bn = ops.gemm_config(M, N, epi, f32)
                    except RuntimeError:
                        assert epi in (ops.EPI_RESID, ops.EPI_RESID_LN)
                        continue
                    assert bn in (64, 128, 256), (epi, f32, M, N, bn)
                    if bn == 256:
                        assert epi == ops.EPI_RESID_LN


def test_throughput_policy_takes_the_wide_tile_for_small_problems(ops):
    """At most 4 row blocks and more than 64 columns: throughput takes 128 (fewest CTAs), latency 64 for a one-row-block
    problem that fits one wave either way.  Neither depends on the SM count beyond the few tiles involved."""
    try:
        for epi in (ops.EPI_BIAS, ops.EPI_RELU, ops.EPI_TABLE, ops.EPI_SWISH, ops.EPI_GELU, ops.EPI_TANH, ops.EPI_RESID):
            ops.set_tile_policy('throughput')
            for M in (1, 300, 512):
                for N in (100, 256, 4234):
                    assert ops.gemm_config(M, N, epi) == 128, (epi, M, N)
            assert ops.gemm_config(513, 100, epi) == 64    # 5 row blocks: the latency cost model applies
            ops.set_tile_policy('latency')
            assert ops.gemm_config(1, 256, epi) == 64
    finally:
        ops.set_tile_policy('latency')


def test_bad_arguments_are_refused(ops):
    for args in ((0, 64, 0, 0), (64, 0, 0, 0), (64, 64, 9, 0), (64, 64, -1, 0)):
        with pytest.raises(RuntimeError, match='otb_gemm_config'):
            ops.gemm_config(*args)
