"""Plain torch restatement of the determinant tail, in fp64 (the reference) or fp32 (the yardstick for what fp32 arithmetic gets
wrong anyway): the orbital matrices A(r, BF) = envelopes (x) activated backflow, their signed log-determinants with
forward-Laplacian jets, and the exp-normalised determinant sum; shared by the Slater-kernel tests.

    A[k][i][mu] = env_k,mu(r_i) mult_act(bf[i][k N + mu]) + g_i add_act(bf_add[i][k N + mu])
    (backflow_transform 'mult': no additive term; 'add': no multiplicative head, mult_act(.) -> 1)
    env_k,mu(r_i) = sum_{m, e} pi[k N + mu][m rep + e] exp(-|zeta[k N + mu][m rep + e]| sqrt(eps + |r_i - R_m|^2))
    g_i = cutoff(r_i) sqrt(sum_{k, mu in i's spin block} env_k,mu(r_i)^2)          (additive branch only)

(reference wf/env.py:57-75, wf/nn_wave_function.py:14-33, :111-171).  The parameter rows [K N][M rep] are the engine's own
layout for every kind: rep = 1 (Psiformer), 3 (TransPsiformer), the largest shell count per nucleus (PauliNet's per-shell
tables, unused terms with pi = 0).  Spin-factorised determinants are the determinants of A with the spin-off-diagonal blocks
zeroed.  Jets: slot t of the r-jet is the unit vector e_t, its Laplacian is 0; the backflow jets are the slot rows."""
import torch

from tc_reference import jet


class TailParams:
    """What the determinant tail reads from an engine: nuclei R [M, 3], envelope tables pi / zeta per spin [K N, M rep], and
    the configuration (n_up, K, full determinants, mult_act, backflow transform, eps of the engine's dtype)."""

    def __init__(self, R, pi_up, pi_dn, zeta_up, zeta_dn, n_up, K, full_det=True, mult_act='identity', transform='mult',
                 eps=2.220446049250313e-16, conf_w=None):
        self.R, self.pi_up, self.pi_dn, self.zeta_up, self.zeta_dn = R, pi_up, pi_dn, zeta_up, zeta_dn
        self.n_up, self.K, self.full_det, self.mult_act, self.transform, self.eps = n_up, K, full_det, mult_act, transform, eps
        self.conf_w = conf_w

    @classmethod
    def of_engine(cls, eng, dtype=torch.float64):
        """The parameters as the device sees them (rounded to fp32 for an fp32 engine)."""
        from tc_reference import weight

        W = lambda n: weight(eng, n, dtype)
        sp = eng.spec
        R = torch.as_tensor(eng.hamil.mol.coords, dtype=eng.dtype).to(dtype)
        return cls(R, W('env.pi_up'), W('env.pi_dn'), W('env.zeta_up'), W('env.zeta_dn'), sp.n_up, sp.n_determinants,
                   sp.full_determinant, sp.mult_act, sp.backflow_transform, torch.finfo(eng.dtype).eps,
                   W('conf.w')[0] if sp.conf_coeff == 'linear' else None)

    def to(self, dtype, device='cpu'):
        c = lambda t: None if t is None else t.to(device, dtype)
        return TailParams(c(self.R), c(self.pi_up), c(self.pi_dn), c(self.zeta_up), c(self.zeta_dn), self.n_up, self.K,
                          self.full_det, self.mult_act, self.transform, self.eps, c(self.conf_w))


def envelopes(r, P):
    """r [B, N, 3] -> env [B, K, N, N] (determinant k, electron i, orbital mu), the spin of electron i picking the table."""
    B, N, _ = r.shape
    M = P.R.shape[0]
    rep = P.pi_up.shape[1] // M
    rho = (P.eps + ((r[:, :, None, :] - P.R[None, None]) ** 2).sum(-1)).sqrt()  # [B, N, M]
    rho = rho.repeat_interleave(rep, dim=-1)                                      # [B, N, M rep]
    out = []
    for pi, ze, sl in ((P.pi_up, P.zeta_up, slice(0, P.n_up)), (P.pi_dn, P.zeta_dn, slice(P.n_up, N))):
        # [B, n_s, K N] = sum_j pi[o, j] exp(-|zeta[o, j]| rho[b, i, j])
        e = (pi[None, None] * torch.exp(-ze.abs()[None, None] * rho[:, sl, None, :])).sum(-1)
        out.append(e)
    env = torch.cat(out, dim=1).reshape(B, N, P.K, N)
    return env.permute(0, 2, 1, 3)


def _spin_mask(N, n_up, like):
    up = torch.arange(N, device=like.device) < n_up
    return (up[:, None] == up[None, :]).to(like.dtype)


def orbitals(r, bf, P):
    """r [B, N, 3], bf [B, N, BFW] (pre-activation head rows) -> A [B, K, N, N]."""
    B, N, _ = r.shape
    KN = P.K * N
    env = envelopes(r, P)
    mask = None if P.full_det else _spin_mask(N, P.n_up, env)
    if mask is not None:
        env = env * mask
    heads = lambda x: x.reshape(B, N, P.K, N).permute(0, 2, 1, 3)
    A = env  # without a multiplicative head the envelopes pass unscaled ('add')
    if P.transform != 'add':
        f = bf[..., :KN]
        A = env * heads(1 + 2 * torch.tanh(f / 4) if P.mult_act == 'default' else f)
    if P.transform != 'mult':
        fa = bf[..., KN:2 * KN] if P.transform == 'both' else bf[..., :KN]
        # g_i = cutoff(r_i) |envelopes of electron i over the determinants and its spin block's orbitals|
        nrm = (env ** 2).sum(dim=(1, 3)).sqrt()                                   # [B, N]
        dist = ((r[:, :, None, :] - P.R[None, None]) ** 2).sum(-1).sqrt().min(-1).values * 2
        cut = torch.where(dist < 1, dist ** 2 * (6 - 8 * dist + 3 * dist ** 2), torch.ones_like(dist))
        add = (cut * nrm)[:, None, :, None] * heads(0.1 * torch.tanh(fa / 4))
        A = A + (add * mask if mask is not None else add)
    return A


def slater_value(r, bf, P):
    """-> (sign [B, K], log|det A| [B, K]) by torch.linalg.slogdet."""
    return torch.linalg.slogdet(orbitals(r, bf, P))


def logabsdet_lu(A):
    """log|det A| as the sum of log|pivot| of an LU elimination in plain tensor ops, the row order of LAPACK's partial
    pivoting taken from the primal matrix.  The value equals slogdet's; it exists for the jets: torch's forward-mode rule of
    slogdet is first-order only (forward over forward gives a wrong second derivative), the elementary ops here nest."""
    Pm = torch.linalg.lu(A.detach())[0]
    U = Pm.transpose(-1, -2) @ A
    out = 0
    for _ in range(A.shape[-1]):
        piv = U[..., 0, 0]
        out = out + torch.log(piv.abs())
        U = U[..., 1:, 1:] - U[..., 1:, :1] * (U[..., :1, 1:] / piv[..., None, None])
    return out


def slater_ref(r, BF, P, S, dtype=torch.float64):
    """Slater determinants of the engine's tail on walkers r [B, N, 3] and slot rows BF [B N S][BFW] (row (b N + i) S + s,
    before activation) -> (sign [B, K], log [B, K], grad [B, K, 3N] or None, lap [B, K] or None); S = 1 or 3N + 2.  Sign and
    log from slogdet; the jets are those of log|det A| (logabsdet_lu) by nested forward-mode AD (tc_reference.jet)."""
    P = P.to(dtype, r.device)
    r = r.to(dtype)
    B, N, _ = r.shape
    bf = BF.to(r.device, dtype).reshape(B, N, S, -1)
    sign, logabs = slater_value(r, bf[:, :, 0], P)
    if S == 1:
        return sign, logabs, None, None
    W = bf.shape[-1]
    T3 = 3 * N
    nr = B * N * 3
    x = torch.cat([r.reshape(-1), bf[:, :, 0].reshape(-1)])
    rt = torch.eye(T3, dtype=dtype, device=r.device).reshape(T3, 1, N * 3).expand(T3, B, N * 3).reshape(T3, nr)
    xt = torch.cat([rt, bf[:, :, 1:S - 1].permute(2, 0, 1, 3).reshape(T3, -1)], dim=1)
    xL = torch.cat([torch.zeros(nr, dtype=dtype, device=r.device), bf[:, :, S - 1].reshape(-1)])
    f = lambda y: logabsdet_lu(orbitals(y[:nr].reshape(B, N, 3), y[nr:].reshape(B, N, W), P))
    _, d1, lap = jet(f, x, xt, xL)
    return sign, logabs, d1.permute(1, 2, 0), lap


def det_sum_ref(det_sign, det_log, det_grad=None, det_lap=None, conf_w=None, dtype=torch.float64):
    """The exp-normalised determinant sum of wf/nn_wave_function.py:152-171 (no cusp, no Jastrow) on det_sign / det_log [B, K]
    -> (sign [B], log|psi| [B], grad [B, 3N] or None, lap [B] or None).  psi = sum_k c_k s_k exp(l_k - shift) with the
    stop-gradient shift max_k l_k (0 where that is not finite); a determinant with s_k = 0 contributes nothing.  Jets: log|psi|
    as a function of the l_k (signs fixed), by nested forward-mode AD."""
    s, l = det_sign.to(dtype), det_log.to(dtype)
    c = s * (conf_w.to(s.device, dtype) if conf_w is not None else 1)
    shift = torch.where(s == 0, torch.full_like(l, -float('inf')), l).max(-1, keepdim=True).values
    l = torch.where(s == 0, torch.zeros_like(l), l)  # exp(-inf) has no jet; its weight is zero anyway
    shift = torch.where(torch.isfinite(shift), shift, torch.zeros_like(shift))

    def logpsi(y):
        return torch.log((c * torch.exp(y - shift)).sum(-1).abs()) + shift[:, 0]

    psi = (c * torch.exp(l - shift)).sum(-1)
    sign = torch.sign(psi)
    if det_grad is None:
        return sign, logpsi(l), None, None
    g = det_grad.to(s.device, dtype).permute(2, 0, 1)  # [3N, B, K]
    lap_in = det_lap.to(s.device, dtype)
    g = torch.where(s[None] == 0, torch.zeros_like(g), g)
    lap_in = torch.where(s == 0, torch.zeros_like(lap_in), lap_in)
    val, d1, lap = jet(logpsi, l, g, lap_in)
    return sign, val, d1.T, lap
