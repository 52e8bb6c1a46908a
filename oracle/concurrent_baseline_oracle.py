"""NumPy restatement of rllab's concurrent-mode sample processing with one LinearFeatureBaseline per agent
(rllab/sandbox/rocky/tf/samplers/batch_ma_sampler.py:64-123, the non-recurrent branch, and the fit at :184-188)
over time-major rollout arrays -- the oracle of ``LinearFeatureBaseline(n_agents=A)``, of
``process_samples_concurrent`` and of the madrl_lfb_*_agents / madrl_*_agents_f32 kernels.

Agent a's rows are the (t, e, a) rows of a rollout; its paths are its (env, episode) segments, in the order
``to_paths`` gives them.  Features, time indices and the fit are oracle.baseline_oracle's.

Two flavours of the baseline list:
  independent  one baseline per agent (``[LinearFeatureBaseline(spec) for _ in agents]``);
  shared       the reference runner's ``[baseline for _ in range(len(env.agents))]`` (runners/rurllab.py:275-276):
               one object listed A times, so agent a >= 1 is predicted with the fit just made on agent a-1, agent 0
               with the previous iteration's fit on agent A-1 (zeros before the first fit).
"""
import numpy as np

from oracle import baseline_oracle as bo
from oracle import postproc_oracle as po


def agent_features(obs, done, obs_before=None, t0=None):
    """[A, T*E, Df] float64: agent a's feature rows in (t, e) order."""
    T, E, A, D = np.shape(obs)
    F = bo.features(obs, done, obs_before, t0)
    return F.reshape(T * E, A, 2 * D + 4).transpose(1, 0, 2)


def agent_path_rows(done):
    """(t*E + e) of an agent's rows in path order (env, episode), and the path lengths.  The same for every
    agent: each agent has one path per (env, episode)."""
    rows, lens = bo.path_rows(done, 1)
    return rows, lens


def fit_agents(F, y, reg_coeff=1e-5):
    """F [A, N, Df], y [A, N] (rows in path order) -> the A rllab fits [A, Df]."""
    return np.stack([bo.fit(F[a], y[a], reg_coeff) for a in range(F.shape[0])])


def concurrent_chain(iterations, shared, discount, gae_lambda, center_adv=True, positive_adv=False,
                     reg_coeff=1e-5, fits=None):
    """Runs process_samples's concurrent branch over consecutive rollouts.

    iterations: dicts with obs [T,E,A,D], done [T,E], rew [T,E,A], optional obs_before [E,A,D] and t0 [E].
    fits: optional list (one [A, Df] per iteration) of coefficients to use as each iteration's fit results
    instead of the oracle's lstsq (to follow a device run whose solver differs in the last digits).
    Returns one dict per iteration: values, advantages (processed), returns [T,E,A] float64, ev [A],
    coeffs_used [A, Df] (what each agent was predicted with), coeffs_fit [A, Df]."""
    out = []
    state = None          # shared: the one object's coefficients; independent: one per agent
    for n, it in enumerate(iterations):
        obs, done = np.asarray(it["obs"]), np.asarray(it["done"])
        T, E, A, D = obs.shape
        Df = 2 * D + 4
        if not shared and state is None:
            state = [None] * A
        F = agent_features(obs, done, it.get("obs_before"), it.get("t0"))
        rows, lens = agent_path_rows(done)
        rew = np.asarray(it["rew"], dtype=np.float64)
        values = np.zeros((T, E, A))
        adv = np.zeros((T, E, A))
        ret = np.zeros((T, E, A))
        ev = np.zeros(A)
        used = np.zeros((A, Df))
        fitted = np.zeros((A, Df))
        obj = state if shared else None
        for a in range(A):
            coef = obj if shared else state[a]
            if coef is not None:
                used[a] = coef
            v = F[a].dot(coef) if coef is not None else np.zeros(T * E)
            values[:, :, a] = v.reshape(T, E)
            for e in range(E):
                ad, rt = po.gae_env(rew[:, e, a:a + 1], values[:, e, a:a + 1], done[:, e], discount, gae_lambda)
                adv[:, e, a], ret[:, e, a] = ad[:, 0], rt[:, 0]
            vp, rp = values[:, :, a].reshape(-1)[rows], ret[:, :, a].reshape(-1)[rows]
            ev[a] = po.explained_variance_1d(vp, rp)
            ap = adv[:, :, a].reshape(-1)[rows]
            if center_adv:
                ap = po.center_advantages(ap)
            if positive_adv:
                ap = po.shift_advantages_to_positive(ap)
            col = np.empty(T * E)
            col[rows] = ap
            adv[:, :, a] = col.reshape(T, E)
            c = bo.fit(F[a][rows], rp, reg_coeff) if fits is None else np.asarray(fits[n][a], dtype=np.float64)
            fitted[a] = c
            if shared:
                obj = c
            else:
                state[a] = c
        if shared:
            state = obj
        out.append(dict(values=values, advantages=adv, returns=ret, ev=ev, coeffs_used=used, coeffs_fit=fitted))
    return out
