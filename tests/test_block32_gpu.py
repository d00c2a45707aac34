"""32-warp blocks of the arm and legged kernel builds (NVP 14, 15, 21, 22; run with -m gpu on an H100).

The per-env scratch of these models is small enough for 32 envs to share one block's shared memory, so a 4096-env Fetch batch
runs as one wave of 128 blocks on 132 SMs.  tests/test_batch_invariance_gpu.py probes block sizes 1..28; this module holds the
32-warp launches to the same rule, with that module's envs, reference launches and comparisons: every env equals the 7-warp
launch of the same envs BIT FOR BIT."""
import ctypes

import pytest
import torch

from tests.test_batch_invariance_gpu import (_assert_same, _backend, _differ, _launch_config, _masks, _needs_cabi, _num_sms, _prepare,
                                             _run_masked, _run_steps)

pytestmark = pytest.mark.gpu

ARM_CASES = ("antmaze", "pointmaze", "fetch_reach", "fetch_pick", "fetch_push", "fetch_slide")
SMEM_MAX = 232448   # dynamic shared memory one block may opt into on sm_90 (227 KB); b200sim_create's fits() adds 64 bytes of slack


@pytest.fixture(params=ARM_CASES)
def arm_case(request, monkeypatch):
    return _prepare(request.param, monkeypatch)


def _smem_words(c, w, mp):
    be = _backend(c, 1, w, mp)
    smem = ctypes.c_int()
    assert be.L.b200sim_launch_config(be.h, ctypes.byref(smem), None, None) == 0
    be.close()
    return smem.value // 4


def test_32_warps_accepted_exactly_when_they_fit(arm_case, monkeypatch):
    """b200sim_create takes B200SIM_WPB=32 exactly when (hot_words + 32 scr_words) * 4 + 64 bytes fit one block; the sizes come
    from the launch configurations at 7 and 8 warps.  Every arm and legged model fits."""
    probe = _backend(arm_case, 1, None, monkeypatch)
    _needs_cabi(probe)
    probe.close()
    s7, s8 = _smem_words(arm_case, 7, monkeypatch), _smem_words(arm_case, 8, monkeypatch)
    scr = s8 - s7
    hot = s7 - 7 * scr
    fits = (hot + 32 * scr) * 4 + 64 <= SMEM_MAX
    try:
        _backend(arm_case, 1, 32, monkeypatch).close()
        accepted = True
    except RuntimeError:
        accepted = False
    assert accepted == fits, f"hot {hot} + 32 x scratch {scr} words: fits {fits}, accepted {accepted}"
    assert fits, f"hot {hot} + 32 x scratch {scr} words no longer fit one block"


def test_32_warps_reproduce_the_reference(arm_case, monkeypatch):
    """All K envs and N = K // 32 * 32 + 1 envs (a tail block with one active warp) at 32 warps per block."""
    ref, S, acts, el0, K = arm_case["ref"], arm_case["S"], arm_case["acts"], arm_case["el0"], arm_case["K"]
    probe = _backend(arm_case, 1, None, monkeypatch)
    _needs_cabi(probe)
    probe.close()
    for n in sorted({K, (K - 1) // 32 * 32 + 1}):
        be = _backend(arm_case, n, 32, monkeypatch)
        got = _run_steps(be, S[:n], [a[:n].contiguous() for a in acts], el0[:n])
        be.close()
        idx = torch.arange(n, device=S.device)
        _assert_same(ref, got, idx, idx, f"32 warps per block, N = {n}")


def test_32_warp_masked_launches(arm_case, monkeypatch):
    """refresh and raw_step_masked at 32 warps per block: unmasked envs equal the unmasked 7-warp launch, masked envs keep their
    state record, output row and step counter."""
    S, el0, K = arm_case["S"], arm_case["el0"], arm_case["K"]
    be = _backend(arm_case, K, 32, monkeypatch)
    _needs_cabi(be)
    S32 = S.view(torch.int32)
    for mname, m in _masks(K, 32, S.device).items():
        for kind in ("refresh", "raw"):
            ref = arm_case["ref_masked"][kind]
            got = _run_masked(be, S, el0, kind, m)
            what = f"{kind}, mask '{mname}', 32 warps per block"
            idx = m.nonzero().flatten()
            bad = _differ(ref["rows"][idx], got["rows"][idx]) + _differ(ref["state"][idx], got["state"][idx])
            assert not bad, f"{what}: active envs {idx[bad[:8]].tolist()} differ from the reference launch"
            idle = (~m).nonzero().flatten()
            bad = _differ(S32[idle], got["state"][idle])
            assert not bad, f"{what}: masked-out envs {idle[bad[:8]].tolist()} had their state record changed"
            assert torch.equal(got["elapsed"], el0), f"{what}: step counters changed"
    be.close()


def test_fetch_4096_runs_in_one_wave(monkeypatch):
    """The default block size of the 4096-env FetchPickAndPlace batch is 32 warps: 128 blocks, no more than one per SM."""
    c = _prepare("fetch_pick", monkeypatch)
    be = _backend(c, 4096, None, monkeypatch)
    _needs_cabi(be)
    w, nb = _launch_config(be)
    be.close()
    assert (w, nb) == (32, 128)
    assert nb <= _num_sms(c["S"].device)
