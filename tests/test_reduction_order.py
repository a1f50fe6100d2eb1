"""The packed warp reductions of kllm_device.cuh (block128_sum_vt_packed, block128_sum_quad_packed)
restated lane by lane in numpy float32 and compared with cub::BlockReduce<float,128>::Sum's order
(cub::WarpReduce's shuffle-down tree, offsets 1, 2, 4, 8, 16, inside each virtual warp, then ((w0 + w1) + w2) + w3 --
matmul_kernel.cu:7-46 / :48-89 as compiled): every addition has the same two operands, so the bits
must agree for ANY input.  The GPU tests pin the kernels against the reference; this pins the
argument the kernels rely on, on CPU, with adversarial magnitudes."""
import numpy as np
import pytest

f32 = np.float32


def cub_block128(v):
    """v[128] = the 128 threads' partial sums, thread t in virtual warp t // 32."""
    warps = []
    for w in range(4):
        x = v[32 * w:32 * w + 32].copy()
        for off in (1, 2, 4, 8, 16):  # shfl_down: lane i += lane i + off (upper lanes pick up garbage, lane 0 never sees it)
            y = x.copy()
            y[:32 - off] = x[:32 - off] + x[off:]
            x = y
        warps.append(x[0])
    return f32(f32(f32(warps[0] + warps[1]) + warps[2]) + warps[3])


def shfl_xor(x, m):
    return x[np.arange(32) ^ m]


def vt_packed(acc):
    """acc[j][lane] = virtual thread lane + 32 j.  Mirrors block128_sum_vt_packed."""
    lane = np.arange(32)
    odd = (lane & 1).astype(bool)
    k0, k1 = np.where(odd, acc[2], acc[0]), np.where(odd, acc[3], acc[1])
    g0, g1 = np.where(odd, acc[0], acc[2]), np.where(odd, acc[1], acc[3])
    s0 = k0 + shfl_xor(g0, 1)
    s1 = k1 + shfl_xor(g1, 1)
    hi = (lane & 2).astype(bool)
    v = np.where(hi, s1, s0) + shfl_xor(np.where(hi, s0, s1), 2)
    for m in (4, 8, 16):
        v = v + shfl_xor(v, m)
    a0, a1, a2, a3 = v[0], v[2], v[1], v[3]
    return f32(f32(f32(a0 + a1) + a2) + a3), v


def quad_packed(acc):
    """acc[e][lane] = virtual thread 4 lane + e.  Mirrors block128_sum_quad_packed."""
    v = (acc[0] + acc[1]) + (acc[2] + acc[3])
    for m in (1, 2, 4):
        v = v + shfl_xor(v, m)
    return f32(f32(f32(v[0] + v[8]) + v[16]) + v[24])


def cases(rng):
    yield rng.standard_normal(128).astype(f32)
    yield (rng.standard_normal(128) * 10.0 ** rng.integers(-20, 20, 128)).astype(f32)  # wild magnitudes
    x = rng.standard_normal(128).astype(f32)
    x[rng.integers(0, 128, 40)] *= f32(1e8)  # cancellation
    yield x - x[::-1].copy()
    yield np.where(rng.random(128) < 0.5, f32(1.0), f32(2.0 ** -24)).astype(f32)  # ties / sticky bits


@pytest.mark.parametrize("seed", range(6))
def test_vt_packed_equals_cub_tree(seed):
    rng = np.random.default_rng(seed)
    for v in cases(rng):
        acc = [v[32 * j:32 * j + 32].copy() for j in range(4)]  # acc[j][lane] = thread lane + 32 j
        got, lanes = vt_packed(acc)
        want = cub_block128(v)
        assert got.tobytes() == want.tobytes()
        # the four virtual-warp sums sit in lanes 0, 2, 1, 3 (mod 4), replicated over the warp
        assert len({lanes[l].tobytes() for l in range(0, 32, 4)}) == 1


@pytest.mark.parametrize("seed", range(6))
def test_quad_packed_equals_cub_tree(seed):
    rng = np.random.default_rng(100 + seed)
    for v in cases(rng):
        acc = [v[e::4].copy() for e in range(4)]  # acc[e][lane] = thread 4 lane + e
        assert quad_packed(acc).tobytes() == cub_block128(v).tobytes()

