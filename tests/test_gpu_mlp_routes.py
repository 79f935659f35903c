"""GPU: which kernels every MLP entry point launches, one case per row of the route in csrc/mlp.cu.

The launches are read by name from a profiler trace: the narrow block kernels (paired or not), the wide pass
kernels at one, two or four K atoms with their <NP, KA>, the K-streamed kernels for O > 128 (float or byte
rows), the FP32 kernels, and whether reduce_partials_kernel runs after the backward (it does not when the
kernel reduces in-kernel).  The IMPALA_MLP_TC / IMPALA_MLP_TCW switches and a misaligned x are covered too.
"""
import re

import numpy as np
import pytest
import torch

from torched_impala_b200 import _cabi, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.fail("GPU test selected but no CUDA device is visible")
    from torched_impala_b200 import ops as _ops

    return _ops


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _ours(name):
    """A kernel of the library's MLP entry points."""
    return "mlp_" in name or "reduce_partials" in name


def _kernel_names(fn, tries=3, reps=3):
    """Names of the kernels fn launches.  A profiler trace can come back without some kernel records of the
    run it covered (several traces in a row have missed the last launch of a call), so it is checked against the
    library's own launch counter.  Every call of fn launches the same kernels, so one trace covers `reps` calls:
    each kernel then has `reps` records, and a trace that misses at most reps - 1 of the library's launches
    still names every kernel fn launches.  A trace that misses more is taken again."""
    lib = _cabi.lib()
    fn()  # first launches (occupancy queries, shared-memory opt-in) stay out of the trace
    torch.cuda.synchronize()
    for _ in range(tries):
        n0 = lib.impala_launch_count()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        launched = lib.impala_launch_count() - n0
        names = [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
        if sum(map(_ours, names)) >= launched - (reps - 1):
            return set(names)
    raise AssertionError(f"{tries} profiler traces missed launches: {sum(map(_ours, names))} of {launched} recorded")


def _has(names, kernel, *targs):
    """A launch of `kernel<targs>` (demangled or mangled name); without targs, any instantiation."""
    if not targs:
        return any(re.search(re.escape(kernel) + "(?![a-z_])", n) for n in names)
    demangled = re.escape(kernel) + "<" + r",\s*".join(map(str, targs)) + ">"
    mangled = re.escape(kernel) + "I" + "".join(f"Li{t}E" for t in targs) + "E"
    return any(re.search(demangled, n) or re.search(mangled, n) for n in names)


# O -> (forward, backward) instantiations at A = 6, H = 256
ROUTES = {24: (("mlp_fwd_tc_kernel", 16, 1), ("mlp_bwd_tcw_kernel", 16, 1)),
          128: (("mlp_fwd_tc_kernel", 16, 4), ("mlp_bwd_tcw_kernel", 32, 4))}


@pytest.mark.parametrize("tensor_cores", ["1", "0"])
@pytest.mark.parametrize("O", sorted(ROUTES))
def test_launches_take_the_16_output_kernels(ops, monkeypatch, O, tensor_cores):
    monkeypatch.setenv("IMPALA_MLP_TC", tensor_cores)
    M, H, N2 = 4096, 256, 6
    rng = np.random.default_rng(O)
    p = ops.pack_params(synth.init_params(1, O, N2, H)["policy"])
    x = dev(rng.standard_normal((M, O), dtype=np.float32))
    dout = dev(rng.standard_normal((M, N2), dtype=np.float32))
    fwd = _kernel_names(lambda: ops.mlp_forward(x, p, O, H, N2))
    bwd = _kernel_names(lambda: ops.mlp_backward(x, p, dout, O, H, N2))
    print(O, tensor_cores, sorted(fwd), sorted(bwd))
    fp32_fwd = any("mlp_fwd_kernel" in n for n in fwd)
    fp32_bwd = any("mlp_bwd_kernel" in n for n in bwd)
    if tensor_cores == "1":
        assert _has(fwd, *ROUTES[O][0]) and not fp32_fwd, fwd
        assert _has(bwd, *ROUTES[O][1]) and not fp32_bwd, bwd
    else:
        assert fp32_fwd and not any("_tc" in n for n in fwd), fwd
        assert fp32_bwd and not any("_tc" in n for n in bwd), bwd


FP32_F, FP32_B, RED = ("mlp_fwd_kernel",), ("mlp_bwd_kernel",), ("reduce_partials_kernel",)
PAIR_F, PAIR_B = ("mlp_fwd_tc_pair_kernel",), ("mlp_bwd_tc_pair_kernel", "false")


def tc_f(np_, ka):
    return ("mlp_fwd_tc_kernel", np_, ka)


def tcw_b(np_, ka):
    return ("mlp_bwd_tcw_kernel", np_, ka)


def obs(np_, xt="float"):
    return [("mlp_fwd_obs_kernel", np_, xt)], [("mlp_bwd_obs_pre_kernel", np_, xt), ("mlp_bwd_obs_dw1_kernel", xt)]


# name: (O, A, H, env, x offset in floats, forward kernels, backward kernels) of the paired entry points
# (impala_mlp_{forward,backward}_pair: the policy with A outputs and the value function on the same rows;
# they call the single entry points unless both networks are on the narrow kernels and 2 <= A <= 4)
OBS_NP32, OBS_NP1 = obs(32), obs(1)
CASES = {
    "c2": (4, 2, 32, {}, 0, [PAIR_F], [FP32_B, RED]),
    "c4": (24, 4, 256, {}, 0, [PAIR_F], [PAIR_B]),
    "c4h512": (24, 4, 512, {}, 0, [tc_f(4, 1), tc_f(1, 1)], [tcw_b(4, 1), tcw_b(1, 1), RED]),
    "c5": (64, 4, 512, {}, 0, [tc_f(4, 2), tc_f(1, 2)], [tcw_b(4, 2), tcw_b(1, 2), RED]),
    "c4a6": (24, 6, 256, {}, 0, [tc_f(16, 1), tc_f(1, 1)], [tcw_b(16, 1), RED, ("mlp_bwd_tc_kernel", 1)]),
    "o32_a20": (32, 20, 256, {}, 0, [tc_f(32, 1), tc_f(1, 1)], [tcw_b(32, 4), tcw_b(1, 1), RED]),
    "o64_a20": (64, 20, 256, {}, 0, [tc_f(32, 2), tc_f(1, 2)], [tcw_b(32, 4), tcw_b(1, 2), RED]),
    "ram": (128, 18, 256, {}, 0, [tc_f(32, 4), tc_f(1, 4)], [tcw_b(32, 4), tcw_b(1, 4), RED]),
    "ram_a6": (128, 6, 256, {}, 0, [tc_f(16, 4), tc_f(1, 4)], [tcw_b(32, 4), tcw_b(1, 4), RED]),
    "ram4": (512, 18, 256, {}, 0, OBS_NP32[0] + OBS_NP1[0], OBS_NP32[1] + OBS_NP1[1] + [RED]),
    "minatar": (400, 6, 256, {}, 0, OBS_NP32[0] + OBS_NP1[0], OBS_NP32[1] + OBS_NP1[1] + [RED]),
    "h96": (24, 4, 96, {}, 0, [PAIR_F], [FP32_B, RED]),
    "o30": (30, 4, 256, {}, 0, [FP32_F], [FP32_B, RED]),
    "c4_x_off1": (24, 4, 256, {}, 1, [FP32_F], [FP32_B, RED]),
    "c4_tc0": (24, 4, 256, {"IMPALA_MLP_TC": "0"}, 0, [FP32_F], [FP32_B, RED]),
    "c5_tc0": (64, 4, 512, {"IMPALA_MLP_TC": "0"}, 0, [FP32_F], [FP32_B, RED]),
    "c4_tcw0": (24, 4, 256, {"IMPALA_MLP_TCW": "0"}, 0, [PAIR_F], [PAIR_B]),
    "c4a6_tcw0": (24, 6, 256, {"IMPALA_MLP_TCW": "0"}, 0, [FP32_F, tc_f(1, 1)],
                  [FP32_B, RED, ("mlp_bwd_tc_kernel", 1)]),
    "c5_tcw0": (64, 4, 512, {"IMPALA_MLP_TCW": "0"}, 0, [FP32_F], [FP32_B, RED]),
}
M = 4096
# shapes impala_mlp_backward_pair_push_supported takes (it sees no pointers, so x alignment is not part of it)
PUSH = {"c4", "c4_x_off1", "c4_tcw0"}


def _check(names, want):
    mine = {n for n in names if _ours(n)}
    for spec in want:
        assert _has(mine, *spec), (spec, sorted(mine))
    stray = [n for n in mine if not any(_has({n}, *spec) for spec in want)]
    assert not stray, (stray, want)


@pytest.mark.parametrize("name", list(CASES))
def test_pair_entry_points_route(ops, monkeypatch, name):
    O, A, H, env, off, want_f, want_b = CASES[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(len(name))
    p = synth.init_params(3, O, A, H)
    p_pi, p_vf = ops.pack_params(p["policy"]), ops.pack_params(p["value_fn"])
    buf = dev(rng.standard_normal(M * O + 4, dtype=np.float32))
    x = buf[off:off + M * O]
    dl = dev(rng.standard_normal((M, A), dtype=np.float32) / M)
    dv = dev(rng.standard_normal(M, dtype=np.float32) / M)
    fwd = _kernel_names(lambda: ops.mlp_forward_pair(x, p_pi, p_vf, M, M, O, H, H, A))
    bwd = _kernel_names(lambda: ops.mlp_backward_pair(x, p_pi, p_vf, dl, dv, O, H, H, A))
    print(name, sorted(fwd), sorted(bwd))
    _check(fwd, want_f)
    _check(bwd, want_b)
    push = _cabi.lib().impala_mlp_backward_pair_push_supported(M, M, O, H, H, A)
    assert push == (name in PUSH), push


@pytest.mark.parametrize("env", [{}, {"IMPALA_MLP_TC": "0"}, {"IMPALA_MLP_TCW": "0"}])
def test_wide_observations_need_the_tensor_cores(ops, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    O, H, N2 = 512, 256, 18
    p = ops.pack_params(synth.init_params(5, O, N2, H)["policy"])
    x = dev(np.zeros((M, O), dtype=np.float32))
    dout = dev(np.zeros((M, N2), dtype=np.float32))
    if env:
        with pytest.raises(_cabi.ImpalaCudaError, match="IMPALA_ERR_UNSUPPORTED_SHAPE"):
            ops.mlp_forward(x, p, O, H, N2)
        assert _cabi.lib().impala_mlp_backward_workspace(M, O, H, N2) == -2
        return
    want_f, want_b = obs(32)
    _check(_kernel_names(lambda: ops.mlp_forward(x, p, O, H, N2)), want_f)
    _check(_kernel_names(lambda: ops.mlp_backward(x, p, dout, O, H, N2)), want_b + [RED])


@pytest.mark.parametrize("O", [128, 512])
def test_byte_entry_points_route(ops, O):
    H, N2 = 256, 18
    rng = np.random.default_rng(O)
    p = ops.pack_params(synth.init_params(7, O, N2, H)["policy"])
    x = dev(rng.integers(0, 256, (M, O), dtype=np.uint8))
    dout = dev(rng.standard_normal((M, N2), dtype=np.float32) / M)
    if O <= 128:
        with pytest.raises(_cabi.ImpalaCudaError):
            ops.mlp_forward_u8(x, p, O, H, N2)
        with pytest.raises(_cabi.ImpalaCudaError):
            ops.mlp_backward_u8(x, p, dout, O, H, N2)
        return
    want_f, want_b = obs(32, "unsigned char")
    _check(_kernel_names(lambda: ops.mlp_forward_u8(x, p, O, H, N2)), want_f)
    _check(_kernel_names(lambda: ops.mlp_backward_u8(x, p, dout, O, H, N2)), want_b + [RED])
