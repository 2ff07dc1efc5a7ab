"""Frozen vectors of the CLOSED-LOOP variant (oracle.es_oracle.ClosedLoopEnvSpec / run_model): there is no reference
implementation of this env (SURVEY.md section 8d names it as an optional synthetic variant), so the oracle is its definition
and these vectors pin the oracle against accidental change.  python tests/golden/make_closed_golden.py -> closed_loop.npz"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import es_oracle as orc  # noqa: E402


def problem():
    obs_dim, act_dim, T = 17, 6, 20
    dims = orc.layer_dims(obs_dim, (64, 64), act_dim)
    P = orc.n_params(dims)
    rs = np.random.RandomState(31)
    table = rs.randn(P + 50_000).astype(np.float32)
    theta = (rs.randn(P) * 0.1).astype(np.float32)
    mean, std = rs.randn(obs_dim) * 0.05, 0.5 + rs.rand(obs_dim)
    return dims, P, table, theta, orc.ClosedLoopEnvSpec(obs_dim, act_dim, T), mean, std


def compute():
    dims, P, table, theta, spec, mean, std = problem()
    out = {}
    for k, idx in enumerate((0, 12345, 49_999)):
        for sgn, sign in enumerate((1.0, -1.0)):
            layers = orc.unflatten(orc.pheno_params(theta, 0.05, sign * orc.table_get(table, idx, P)), dims)
            rews, behv, obs, step = orc.run_model(spec, layers, mean, std, 0.4, spec.T)
            out[f'rews_{k}_{sgn}'] = np.array(rews)
            out[f'pos_{k}_{sgn}'] = np.array(behv[-3:])
            out[f'obs_last_{k}_{sgn}'] = obs[-1]
    pos, neg, inds, steps, obstat = orc.es_test_params(table, theta, 0.05, dims, spec, [900, 901], 3, mean, std, 0.4, spec.T,
                                                       coins_per_eval=1, save_obs_chance=0.5)
    out.update(gen_pos=pos, gen_neg=neg, gen_inds=inds, gen_steps=np.array(steps), ob_sum=obstat.sum, ob_sumsq=obstat.sumsq,
               ob_count=np.array(obstat.count), env_a=spec.env_a, env_b=spec.env_b)
    return out


if __name__ == '__main__':
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'closed_loop.npz')
    np.savez_compressed(path, **compute())
    print(path)
