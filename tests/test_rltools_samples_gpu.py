"""rltools' sample processing on the device (madrl_b200.rltools_sampler) against the golden written by the
reference's own Sampler.process and LinearFeatureBaseline (oracle/make_rltools_golden.py) and the NumPy oracle, in
every control mode, replayed in the training loop's order: the iteration-0 extra batch updates the baselines'
obsnorm and the reward normaliser, then each rollout is processed and the reward normaliser updated."""
import os

import numpy as np
import pytest
import torch

import sharded_edges as se
from oracle import rltools_oracle as ro

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "rltools_samples_ref.npz")
MODES = ("decentralized", "concurrent", "centralized", "zero")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _close(got, want, what):
    scale = max(1e-5 * float(np.max(np.abs(want))), 1e-30)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=scale, err_msg=what)


def _ulps(got, want):
    g, w = np.asarray(got, np.float32).view(np.int32), np.asarray(want, np.float32).view(np.int32)
    return int(np.max(np.abs(g.astype(np.int64) - w.astype(np.int64))))


def _replay_device(settings, rollouts, mode, dtype):
    return se.replay_device(settings, rollouts, mode, dtype)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", ("ragged", "plain"))
def test_process_samples_matches_the_reference(golden, case, mode):
    settings, rollouts = ro.golden_case(golden, case)
    dtype = torch.bfloat16 if case == "plain" else torch.float32
    runs = zip(ro.replay(settings, rollouts, mode), _replay_device(settings, rollouts, mode, dtype))
    A = rollouts[0]["obs"].shape[2]
    pm = "decentralized" if mode == "zero" else mode
    for (k, res, obls, orn), (_, out, bl, rn) in runs:
        key = "%s/%s/r%d/" % (case, mode, k)
        if out is not None:
            done = rollouts[k]["done"]
            nb = A if pm == "concurrent" else 1
            gq = [golden[key + ("a%d/" % b if pm == "concurrent" else "") + "q"] for b in range(nb)]
            ga = [golden[key + ("a%d/" % b if pm == "concurrent" else "") + "adv"] for b in range(nb)]
            split = lambda flat, b: np.split(flat, np.cumsum([len(x) for x in res[b]["q"]])[:-1])  # noqa: E731
            want_q = ro.to_rollout([split(gq[b], b) for b in range(nb)], done, A, pm)
            want_adv = ro.to_rollout([split(ga[b], b) for b in range(nb)], done, A, pm)
            want_v = ro.to_rollout([r["v"] for r in res], done, A, pm)
            _close(out["q"].cpu().numpy(), want_q, key + "q")
            _close(out["advantages"].cpu().numpy(), want_adv, key + "advantages")
            _close(out["values"].cpu().numpy(), want_v, key + "values")
            for b in range(nb):
                st = golden[key + ("a%d/" % b if pm == "concurrent" else "") + "stats"]
                pick = (lambda x: x[b]) if pm == "concurrent" else (lambda x: x)                    # noqa: E731
                assert abs(pick(out["v_r"]) - st[0]) < 1e-6, (key, b)
                assert abs(pick(out["tv_r"]) - st[1]) < 1e-6, (key, b)
                assert pick(out["fallback"]) == bool(st[2]), (key, b)
            if bl is not None:
                w = bl.get_param_values()[0]
                for b in range(nb):
                    gw = golden[key + ("a%d/" % b if pm == "concurrent" else "") + "w"]
                    wb = w[b] if pm == "concurrent" else w
                    np.testing.assert_allclose(wb, gw, rtol=1e-4, atol=1e-6 * np.max(np.abs(gw)), err_msg=key)
        if bl is not None and settings["obsnorm"]:
            cnt, mean, meansq = bl.obsnorm.get_param_values()
            for b, obl in enumerate(obls):
                g = golden[key + ("a%d/" % b if pm == "concurrent" else "") + "obsnorm"].astype(np.float32)
                D = (len(g) - 1) // 2
                pick = (lambda x: x[b]) if pm == "concurrent" else (lambda x: x)                        # noqa: E731
                assert float(pick(cnt)) == g[0]
                assert _ulps(pick(mean), g[1:1 + D]) <= 1 and _ulps(pick(meansq), g[1 + D:]) <= 1, key
        if rn is not None:
            g = golden[key + "rewnorm"].astype(np.float32)
            cnt, mean, meansq = rn.get_param_values()
            assert float(cnt) == g[0] and _ulps(mean, g[1:2]) <= 1 and _ulps(meansq, g[2:3]) <= 1, key


@pytest.mark.parametrize("per_agent", (False, True))
def test_time_baseline_bins_and_reruns(per_agent):
    """Counts exact and sums at 1e-12 against NumPy on the device's own q, t0 shifting first paths, NaN-free, and
    a re-run bit-identical."""
    from madrl_b200 import rltools_sampler as rs
    T, E, A = 37, 301, 3
    g = np.random.RandomState(5)
    done = (g.rand(T, E) < 0.08).astype(np.uint8)
    done[:, 7] = 0
    done[0, 8] = done[T - 1, 9] = 1
    q = g.randn(T, E, A).astype(np.float32)
    t0 = g.randint(0, 20, E).astype(np.int32)
    dev = torch.device("cuda")
    qd, dd, td = (torch.from_numpy(x).to(dev) for x in (q, done, t0))
    simplev, s, c = rs.time_baseline(qd, dd, td, per_agent)
    s2 = rs.time_baseline(qd, dd, td, per_agent)
    assert all(torch.equal(x, y) for x, y in zip((simplev, s, c), s2))
    idx = np.zeros((T, E), np.int64)
    for e in range(E):
        st = 0
        for t in range(T):
            idx[t, e] = t - st + (t0[e] if st == 0 else 0)
            if done[t, e]:
                st = t + 1
    G, L = (A if per_agent else 1), int(idx.max()) + 1
    ws, wc = np.zeros((G, L)), np.zeros((G, L), np.int64)
    for a in range(A):
        np.add.at(ws[a if per_agent else 0], idx, q[..., a].astype(np.float64))
        np.add.at(wc[a if per_agent else 0], idx, 1)
    assert np.array_equal(c.cpu().numpy(), wc)
    np.testing.assert_allclose(s.cpu().numpy(), ws, rtol=1e-12, atol=1e-12)
    want = np.stack([(ws / np.maximum(wc, 1))[a if per_agent else 0][idx] for a in range(A)], -1)
    np.testing.assert_allclose(simplev.cpu().numpy(), want, rtol=1e-6, atol=1e-6)


def test_gram_against_the_oracle_and_rerun(golden):
    """rltools' normal equations with obsnorm, per agent, within 1e-12 sqrt(G_ii G_jj) of NumPy's, bit-identical
    on a re-run."""
    from madrl_b200 import rltools_sampler as rs
    T, E, A, D = 50, 64, 3, 70                      # the observation block crosses a 64-column tile
    g = np.random.RandomState(9)
    obs = (g.randn(T, E, A, D) * 3 + 1).astype(np.float32)
    done = (g.rand(T, E) < 0.05).astype(np.uint8)
    q = g.randn(T, E, A).astype(np.float32)
    dev = torch.device("cuda")
    bl = rs.LinearFeatureBaseline(D, dev, True, n_agents=A)
    od, dd, qd = (torch.from_numpy(x).to(dev) for x in (obs, done, q))
    bl.update_obsnorm(od)
    G = bl.normal_equations(od, dd, qd).cpu().numpy()
    assert np.array_equal(G, bl.normal_equations(od, dd, qd).cpu().numpy())
    cnt, mean, meansq = bl.obsnorm.get_param_values()
    for a in range(A):
        obl = ro.Baseline(D, True)
        obl.obsnorm.count, obl.obsnorm.mean, obl.obsnorm.meansq = cnt[a:a + 1], mean[a][None], meansq[a][None]
        paths = [p for p in ro.batches(obs, q.astype(np.float64), done, None, "concurrent")[a]]
        qs = np.concatenate([p["rewards"] for p in paths])
        want = obl.normal_equations(paths, qs)
        d = np.sqrt(np.abs(np.diag(want)))
        assert np.all(np.abs(G[a] - want) <= 1e-12 * np.outer(d, d) + 1e-300), a


@pytest.mark.parametrize("mode", ("decentralized", "concurrent", "centralized"))
def test_large_rollout_against_pytorch(mode):
    """A C2-sized rollout (T 256, E 2048, A 5, D 32) through two process_samples calls with an obsnorm and a reward
    normaliser, the second one predicting with the first one's fit: q, advantages, values, simplev, v_r, tv_r, the
    fallback and the new coefficients against the PyTorch implementation of oracle/rltools_oracle.py; a re-run of
    each device pass gives the same bits."""
    from madrl_b200 import rltools_sampler as rs
    T, E, A, D = 256, 2048, 5, 32
    g = torch.Generator(device="cuda").manual_seed(3)
    dev = torch.device("cuda")
    obs = torch.randn(T, E, A, D, device=dev, generator=g) * 2 + 0.5
    ob = torch.randn(E, A, D, device=dev, generator=g)
    done = (torch.rand(T, E, device=dev, generator=g) < 0.01).to(torch.uint8)
    rew = obs[..., 0] - 0.5 * obs[..., 1] + torch.randn(T, E, A, device=dev, generator=g)
    if mode == "centralized":
        rew = rew[..., :1].expand(T, E, A).contiguous()
    cen = mode == "centralized"
    vo = obs.reshape(T, E, 1, A * D) if cen else obs
    vb = ob.reshape(E, 1, A * D) if cen else ob
    vr = rew[..., :1] if cen else rew
    bl = rs.LinearFeatureBaseline(vo.shape[-1], dev, True, n_agents=A if mode == "concurrent" else None)
    rn = rs.RunningStandardizer(1, dev)
    bl.update_obsnorm(vo, vb)
    s1 = rn._sums(vr.unsqueeze(-1), None, 1)[0]
    rn.update(vr.unsqueeze(-1))
    assert torch.equal(s1, rn._sums(vr.unsqueeze(-1), None, 1)[0])
    rs.process_samples(bl, obs, done, rew, 0.99, 0.97, rn, mode, obs_before=ob)
    w = bl._coeffs.clone()
    norm = bl.obsnorm.norm_table
    norm = norm if norm.dim() == 3 else norm.unsqueeze(0)
    out = rs.process_samples(bl, obs, done, rew, 0.99, 0.97, rn, mode, obs_before=ob)
    want = ro.torch_process_samples(vo, vb, done, vr, 0.99, 0.97, rn.denom, w, norm, mode == "concurrent")
    for k, kd in (("q", "q"), ("advantages", "adv"), ("values", "values")):
        _close(out[k].cpu().numpy(), want[kd].cpu().numpy(), mode + " " + k)
    simplev = rs.time_baseline(out["q"], done, None, mode == "concurrent")[0]
    _close(simplev.cpu().numpy(), want["simplev"].cpu().numpy(), mode + " simplev")
    pick = (lambda x: list(x)) if mode == "concurrent" else (lambda x: [x])                       # noqa: E731
    assert np.allclose(pick(out["v_r"]), want["v_r"].cpu().numpy().reshape(-1), atol=1e-6)
    assert np.allclose(pick(out["tv_r"]), want["tv_r"].cpu().numpy().reshape(-1), atol=1e-6)
    assert pick(out["fallback"]) == [bool(x) for x in want["fallback"].cpu().numpy().reshape(-1)]
    wn = want["w"].cpu().numpy()
    np.testing.assert_allclose(bl.get_param_values()[0], wn, rtol=1e-6, atol=1e-8 * np.abs(wn).max())
    # re-runs: same inputs, same bits (the baseline's fit would change its state, so it is left out here)
    again = rs.process_samples(None, obs, done, rew, 0.99, 0.97, rn, mode, obs_before=ob)
    once = rs.process_samples(None, obs, done, rew, 0.99, 0.97, rn, mode, obs_before=ob)
    for k in ("q", "advantages", "values"):
        assert torch.equal(again[k], once[k]), k
    assert again["v_r"] == once["v_r"] and again["tv_r"] == once["tv_r"]


@pytest.mark.parametrize("mode", ("decentralized", "concurrent", "centralized"))
@pytest.mark.parametrize("case", ("ragged", "plain"))
def test_sample_fields_match_the_reference(golden, case, mode):
    """The fields serial.py's samplers log, against the oracle's restatement of them on the golden rollouts."""
    from madrl_b200 import rltools_sampler as rs
    _, rollouts = ro.golden_case(golden, case)
    for it in rollouts:
        rew = it["rew_cent"] if mode == "centralized" else it["rew"]
        want = ro.sample_fields(ro.batches(it["obs"], rew.astype(np.float64), it["done"], None, mode))
        got = rs.sample_fields(torch.from_numpy(rew).cuda(), torch.from_numpy(it["done"]).cuda(), mode)
        assert set(got) == set(want)
        for k in ("batch", "avglen", "maxlen", "minlen"):
            assert got[k] == want[k], k
        for k in ("ret", "ravg"):
            assert abs(got[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])), k
