"""PointInfoNCE (`pcb_nce_forward_backward`, both paths) and the hardest-negative search (`pcb_pdist_rowmin`) against fp64, element by
element, on exactly representable features (tests/exact_loss.py) at every tile, split and chunk edge, with worst-case error bounds.

`pcb_pdist_rowmin` is exact on these operands: minval must equal fp32 sqrt(d2 + 1e-7) bit for bit and argmin the smallest tied index.

PointInfoNCE: the logits are exact, so what remains is the fp32 arithmetic after them.  The bounds below are worst cases of that
arithmetic, derived from the kernels' code; nothing in them is fitted to observed errors.

Derivation
----------
u = 2^-24.  fl(x op y) = (x op y)(1 + d), |d| <= u; contracted multiply-adds (nvcc contracts by default) round once, which only
removes roundings from the chains counted below.  exp2f and expf are within 2 ulp (relative 2^-22 = RHO) and return exactly 1 at 0,
logf is within 1 ulp (2^-23 |result|), sqrtf is correctly rounded (no fast-math).  A positive relative error x is written as a factor
exp(+-lam(x)), lam(x) = -log(1 - x).  The reference logit is z_ij = S_ij / T with S = q k^T exact in fp64; the kernel's logit
sv_ij = fl(S_ij inv_T) (inv_T: the fp32 argument) is within e_ij = u |z_ij| of it.  In the production case (last test) S is not
exact, and e_ij grows by inv_T eps_ij, eps_ij = |S_tc - S| + (3D + 2 (3D / 16)) 2^-23 sum|products| (S_tc: the exact sum of the three
fp16 plane products the tensor cores add).  The second term models the fp32 accumulation of the 3D / 16 K16 MMAs, whose order is not
documented, as truncating: each of the 3D products, and in each MMA the accumulator taken in as an addend and the renormalised result,
may lose less than one unit in the 24th bit of a magnitude no larger than sum|products|.  e_ij also grows by |z_ij| |inv_T T - 1| for
the fp32 rounding of 1/T.

LSE pass, tensor cores (nce_wgmma.cu MODE_LSE).  Row i, split s of tps tiles, column half h: C = 4 tps chunks of 16 columns.
  Chunk: add = sum of exp2f(fl(fl(sv_j - mn) L2E)) over the chunk's valid columns; the argument is (sv_j - mn) log2(e) (1 + eta),
  eta = (1 + u)^2 (1 + |fl32(log2 e) / log2 e - 1|) - 1, so the term is e^(sv_j - mn) exp(+-|sv_j - mn| eta) exp(+-lam(RHO)).
  Running value: l = l exp2f(fl(fl(m_old - mn) L2E)) + add at each later chunk, then the two halves, then the split combine
  l = sum_s l_s expf(fl(m_s - m)).  The arguments of the successive exponentials of one term telescope: their magnitudes add up to
  m_i - sv_j, so their eta errors add up to (m_i - sv_j) eta; the combine's expf has a smaller argument error (u) and is covered.
  Per term at most N_exp = 1 + (C - 1) + 1 + 1 = C + 2 exponentials and N_rnd = 15 (the chunk sum) + 2 (C - 1) (rescale, add) + 2
  (half combine) + S (split combine: one product, S - 1 sums) roundings, all of positive quantities.  Hence l_c = sum_j
  e^(sv_j - m) f_j with |log f_j| <= (m - sv_j) eta + N_exp lam(RHO) + N_rnd lam(u), and with m - sv_j <= zmax - z_j + e_max + e_j
      |log(l_c e^m) - lse_i| <= B_i = log sum_j w_ij exp(a_ij),  a_ij = e_ij + (zmax_i - z_ij + e_max_i + e_ij) eta + N_exp lam(RHO)
                                                                        + N_rnd lam(u),    w_ij = softmax(z_i)_j
  (a weighted mean of factors within exp(+-a_ij)), plus n 2^-140 for exponentials that underflow into subnormals (2 ulp absolute).
  lse_c = fl(m + logf(l_c)):  E_lse_i = E2 + u (|lse_i| + E2),  E2 = B_i + 2^-23 (lse_i - zmax_i + e_max_i + B_i).
  SIMT (loss.cu nce_softmax_kernel): one expf per term, argument error u (eta = u), N_exp = 1, N_rnd = ceil(n / 256) - 1 (a thread's
  column stride) + 5 (warp tree) + 7 (the 8 warp sums).
  rowloss_i = fl(lse_c - sv_ii):  E_row_i = E_lse_i + e_ii + u (|rowloss_i| + E_lse_i + e_ii).
  loss = fl32(fp64 mean):  E_loss = E_m + u (|loss| + E_m),  E_m = mean E_row + (n + 16) 2^-53 mean(|rowloss| + E_row).

Gradient passes.  P_ij = exp(z_ij - lse_i).  The kernel's p_ij = exp2f(fl(fl(sv_ij - lse_c_i) L2E)) (SIMT: expf(fl(sv - lse_c)))
has |log(p / P)| <= b_ij = e_ij + E_lse_i + (lse_i - z_ij + e_ij + E_lse_i) eta + lam(RHO), so |p - P| <= dP = P expm1(b) + 2^-148.
  Tensor cores, dq_i = (sum_j p_ij k_j - k_i) scale, scale = fl(inv_T / n): every term goes through at most K = 64 tps (its half's
  fused multiply-adds) + 1 (half combine) + S - 1 (split sum) roundings, so with gamma_K = K u / (1 - K u)
      |sum_c - sum_j P_ij k_jd| <= E_s = sum_j dP_ij |k_jd| + gamma_K sum_j (P_ij + dP_ij) |k_jd|
      |dq_c - dq| <= (inv_T / n) (E_s + gamma_3 (|G_id| + E_s)),   G_id = sum_j P_ij k_jd - k_id   (subtract, scale, multiply)
  and dk the same with the roles of q and k swapped (the column pass reuses p_ij and lse_c of the row).
  SIMT, G_c = fl(fl(p - delta) scale) is within dG = (inv_T / n)(dP + gamma_3 (|P - delta| + dP)) of G = (P - delta) inv_T / n, and
  the sgemm's K = n chain adds gamma_n sum_j |G_c| |k_jd|:  |dq_c - dq| <= sum_j dG_ij |k_jd| + gamma_n sum_j |G_c_ij| |k_jd|.
The fp64 reference itself is allowed 2^-36 of the magnitudes it sums (n 2^-53 with room to spare).
"""
import math

import numpy as np
import pytest
import torch

from tests import exact_loss as X

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RHO = 2.0 ** -22                     # exp2f / expf: 2 ulp
LOGF = 2.0 ** -23                    # logf: 1 ulp
REF = 2.0 ** -36                     # the fp64 reference
L2E_ERR = abs(float(np.float32(1.4426950408889634)) * math.log(2.0) - 1.0)
ETA_TC = (1 + U) ** 2 * (1 + L2E_ERR) - 1
BLOCK = 1 << 22                      # reference elements per row block: peak device memory well below 2 GB at n = 128 SMs + 1
F64 = torch.float64


def tc_acc_steps(D):
    """Truncating steps of one tensor-core dot product of width D (see the derivation): 3D products, 2 per K16 MMA."""
    return 3 * D + 2 * (3 * D // 16)


def lam(x):
    return -math.log1p(-x)


def gamma(k):
    return k * U / (1 - k * U)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _chain(path, n, geo):
    """(N_exp, N_rnd, eta, K) of the derivation for one call."""
    if path == "tc":
        _, splits, tps = geo
        C = 4 * tps
        return C + 2, 15 + 2 * (C - 1) + 2 + splits, ETA_TC, 64 * tps + splits
    return 1, max(-(-n // 256) - 1, 0) + 12, U, n


def nce_reference(q, k, inv_T, path, geo, inv_T_ref=None, eps=None):
    """fp64 loss, dq, dk and their bounds (see the derivation).  q, k: fp64 [n, D] on the device (the fp32 values the kernel reads);
    inv_T: the kernel's fp32 1/T; inv_T_ref: the reference's 1/T (default inv_T); eps(r0, r1): bound on |S_c - S| for rows r0:r1."""
    n, D = q.shape
    itr = inv_T if inv_T_ref is None else inv_T_ref
    d_inv = abs(inv_T - itr)
    n_exp, n_rnd, eta, K = _chain(path, n, geo)
    const = n_exp * lam(RHO) + n_rnd * lam(U)
    R = max(1, BLOCK // n)
    aq, ak = q.abs(), k.abs()
    lse, E_lse, rowloss, E_row = (torch.empty(n, dtype=F64, device=q.device) for _ in range(4))
    zmax_all = -math.inf

    def logits(r0, r1):
        S = q[r0:r1] @ k.T
        z = S * itr
        e = U * z.abs() if eps is None else inv_T * eps(r0, r1) * (1 + U) + S.abs() * (d_inv + U * inv_T)
        return z, e

    for r0 in range(0, n, R):
        r1 = min(n, r0 + R)
        z, e = logits(r0, r1)
        zmax, emax = z.max(1).values, e.max(1).values
        zmax_all = max(zmax_all, float(zmax.max()))
        ls = torch.logsumexp(z, 1)
        a = e + (zmax[:, None] - z + emax[:, None] + e) * eta + const
        B = torch.logsumexp(z - ls[:, None] + a, 1) + n * 2.0 ** -140
        E2 = B + LOGF * (ls - zmax + emax + B)
        El = E2 + U * (ls.abs() + E2) + REF * (1 + ls.abs())
        i = torch.arange(r1 - r0, device=q.device)
        zii, eii = z[i, i + r0], e[i, i + r0]
        rl = ls - zii
        lse[r0:r1], E_lse[r0:r1], rowloss[r0:r1] = ls, El, rl
        E_row[r0:r1] = El + eii + U * (rl.abs() + El + eii)
    loss = float(rowloss.mean())
    E_m = float(E_row.mean()) + (n + 16) * 2.0 ** -53 * float((rowloss.abs() + E_row).mean())
    E_loss = E_m + U * (abs(loss) + E_m) + REF * (1 + abs(loss))

    s_ref, s_ker = itr / n, inv_T / n
    g3, gK = gamma(3), gamma(K)
    dq, E_dq = torch.empty_like(q), torch.empty_like(q)
    Tk = [torch.zeros_like(k) for _ in range(4)]          # dk: sum_i P q_i, and the three magnitude sums over i
    for r0 in range(0, n, R):
        r1 = min(n, r0 + R)
        z, e = logits(r0, r1)
        l, El = lse[r0:r1, None], E_lse[r0:r1, None]
        P = torch.exp(z - l)
        b = e + El + (l - z + e + El) * eta + lam(RHO)
        dP = P * torch.expm1(b) + 2.0 ** -148
        i = torch.arange(r1 - r0, device=q.device)
        if path == "tc":
            G = P @ k - k[r0:r1]
            Es = dP @ ak + gK * ((P + dP) @ ak)
            dq[r0:r1] = G * s_ref
            E_dq[r0:r1] = s_ker * (Es + g3 * (G.abs() + Es)) + d_inv / n * (G.abs() + Es) + REF * s_ref * (P @ ak + ak[r0:r1])
            Tk[0] += P.T @ q[r0:r1]; Tk[1] += dP.T @ aq[r0:r1]; Tk[2] += (P + dP).T @ aq[r0:r1]; Tk[3] += P.T @ aq[r0:r1]
        else:
            Pm = P.clone()
            Pm[i, i + r0] -= 1
            dG = s_ker * (dP + g3 * (Pm.abs() + dP)) + d_inv / n * Pm.abs()
            Gc = s_ker * (Pm.abs() + dP) * (1 + g3)
            dq[r0:r1] = (Pm @ k) * s_ref
            E_dq[r0:r1] = dG @ ak + gamma(n) * (Gc @ ak) + REF * s_ref * (Pm.abs() @ ak)
            Tk[0] += Pm.T @ q[r0:r1]; Tk[1] += dG.T @ aq[r0:r1]; Tk[2] += Gc.T @ aq[r0:r1]; Tk[3] += Pm.abs().T @ aq[r0:r1]
    if path == "tc":
        G = Tk[0] - q
        Es = Tk[1] + gK * Tk[2]
        dk = G * s_ref
        E_dk = s_ker * (Es + g3 * (G.abs() + Es)) + d_inv / n * (G.abs() + Es) + REF * s_ref * (Tk[3] + aq)
    else:
        dk = Tk[0] * s_ref
        E_dk = Tk[1] + gamma(n) * Tk[2] + REF * s_ref * Tk[3]
    return dict(loss=loss, E_loss=E_loss, dq=dq, E_dq=E_dq, dk=dk, E_dk=E_dk, zmax=zmax_all)


def nce_call(q, k, inv_T):
    """pcb_nce_forward_backward on fp32 q, k with a workspace and outputs full of NaN (an unwritten entry cannot pass)."""
    from pointcontrast_b200 import _lib
    n, D = q.shape
    loss = torch.full((), float("nan"), device="cuda")
    dq, dk = torch.full_like(q, float("nan")), torch.full_like(k, float("nan"))
    wsb = _lib.lib.pcb_nce_ws_bytes(n)
    ws = torch.full((wsb,), 0xFF, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib.pcb_nce_forward_backward(_lib.ptr(q), _lib.ptr(k), n, D, inv_T, _lib.ptr(loss), _lib.ptr(dq), _lib.ptr(dk),
                                                 _lib.ptr(ws), wsb, _lib.stream()))
    torch.cuda.synchronize()
    return loss, dq, dk


# (path, output) -> the element closest to its bound over every case run: (|error| / bound, |error|, bound, case), and the largest
# |error| of any element; printed at the end of the module (pytest -s)
_REPORT = {}


def _note(key, case, got, ref, bound):
    got, ref, bound = (torch.as_tensor(t, dtype=F64).flatten().cpu() for t in (got, ref, bound))
    err = (got - ref).abs()
    ratio = torch.where(err > 0, err / bound, 0.0)
    i = int(ratio.argmax())
    old = _REPORT.get(key, (-1.0, 0.0, 0.0, None, 0.0))
    worst = (float(ratio[i]), float(err[i]), float(bound[i]), case) if float(ratio[i]) > old[0] else old[:4]
    _REPORT[key] = worst + (max(old[4], float(err.max())),)


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    if _REPORT:
        print(f"\nworst error against its bound on {torch.cuda.get_device_properties(0).name}, {_sms()} SMs")
        for (path, out), (ratio, err, bound, case, emax) in sorted(_REPORT.items()):
            print(f"  {path:>10} {out:>4}: |err| {err:.3e} <= bound {bound:.3e} (ratio {ratio:.3f}) at {case}; largest |err| {emax:.3e}")


def check_nce(pattern, T, n, D, seed, path, geo):
    """One case: the kernel against the fp64 reference, every output element within its bound.  Returns the kernel's outputs."""
    q, k = X.nce_operands(pattern, n, D, seed)
    inv_T = float(np.float32(1.0 / T))
    qc, kc = q.cuda(), k.cuda()
    loss, dq, dk = nce_call(qc, kc, inv_T)
    r = nce_reference(qc.double(), kc.double(), inv_T, path, geo)
    if pattern == "negative":
        assert r["zmax"] <= -0.5, r["zmax"]          # a zero-filled padding column would be the largest logit of every row
    tag = (pattern, T, n, D, path)
    el = abs(float(loss) - r["loss"])
    assert el <= r["E_loss"], (tag, "loss", float(loss), r["loss"], r["E_loss"])
    _note((path, "loss"), tag, float(loss), r["loss"], r["E_loss"])
    for name, got in (("dq", dq), ("dk", dk)):
        ok = (got.double() - r[name]).abs() <= r["E_" + name]
        if not bool(ok.all()):
            bad = torch.nonzero(~ok)[0].tolist()
            raise AssertionError((tag, name, bad, float(got[tuple(bad)]), float(r[name][tuple(bad)]), float(r["E_" + name][tuple(bad)])))
        _note((path, name), tag, got, r[name], r["E_" + name])
    return loss, dq, dk


def _run_shape(path, n, D, geo):
    for ci, (pattern, T) in enumerate(X.NCE_CASES):
        seed = X.nce_seed(D, n, ci)
        outs = check_nce(pattern, T, n, D, seed, path, geo)
        if ci == 0:              # determinism: a second call gives the same bits
            again = nce_call(*(t.cuda() for t in X.nce_operands(pattern, n, D, seed)), float(np.float32(1.0 / T)))
            for a, b in zip(outs, again):
                assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_case_matrix_reaches_every_split_geometry_on_this_device():
    sms = _sms()
    seen = set().union(*(X.nce_reaches(X.tc_size(n, sms), sms) for n in X.TC_N))
    assert seen >= {"partial last tile", "single split of several tiles", "several splits", "short last split",
                    "diagonal in half 0 of a split's last tile", "diagonal in half 1 of a split's last tile"}, (sms, seen)


@pytest.mark.parametrize("D", X.TC_D)
@pytest.mark.parametrize("n", X.TC_N)
def test_nce_tensor_core_path_within_worst_case_bounds(n, D):
    sms = _sms()
    n = X.tc_size(n, sms)
    _run_shape("tc", n, D, X.nce_geometry(n, sms))


@pytest.mark.parametrize("D", X.SIMT_D)
@pytest.mark.parametrize("n", X.SIMT_N)
def test_nce_simt_path_within_worst_case_bounds(n, D):
    _run_shape("simt", n, D, None)


def test_point_nce_production_call_within_worst_case_bounds():
    """losses.point_nce_loss as the PointInfoNCE trainer calls it (n = 4096, T = 0.07, D = 32, repeated keys) on L2-normalised
    features, against oracle/loss_cpu.py in fp64."""
    from oracle import loss_cpu
    from pointcontrast_b200 import losses
    n, T, D = 4096, 0.07, 32
    g = torch.Generator().manual_seed(4096)
    N0, N1 = 3 * n, 3 * n + 11
    F0 = torch.nn.functional.normalize(torch.randn(N0, D, generator=g, dtype=F64), dim=1)
    F1 = torch.nn.functional.normalize(torch.randn(N1, D, generator=g, dtype=F64), dim=1)
    q_rows = torch.randperm(N0, generator=g)[:n]
    k_rows = torch.randint(0, N1, (n,), generator=g)
    first = torch.from_numpy(np.unique(k_rows.numpy(), return_index=True)[1])     # one write per key row: reproducible features
    F1[k_rows[first]] = torch.nn.functional.normalize(F1[k_rows[first]] + F0[q_rows[first]], dim=1)
    F0, F1 = F0.float(), F1.float()
    assert len(torch.unique(k_rows)) < n
    f0, f1 = F0.cuda().requires_grad_(True), F1.cuda().requires_grad_(True)
    l = losses.point_nce_loss(f0, f1, q_rows.cuda(), k_rows.cuda(), T)
    l.backward()
    f0o, f1o = F0.double().requires_grad_(True), F1.double().requires_grad_(True)
    lo = loss_cpu.point_nce_loss(f0o, f1o, q_rows, k_rows, T)
    lo.backward()

    q, k = F0.double()[q_rows].cuda(), F1.double()[k_rows].cuda()
    planes = []
    for x in (q, k):
        hi = x.float().half()
        planes.append((hi.double(), (x.float() - hi.float()).half().double()))
    (hq, lq), (hk, lk) = planes

    def eps(r0, r1):
        S = q[r0:r1] @ k.T
        Stc = hq[r0:r1] @ hk.T + hq[r0:r1] @ lk.T + lq[r0:r1] @ hk.T
        mag = hq[r0:r1].abs() @ hk.abs().T + hq[r0:r1].abs() @ lk.abs().T + lq[r0:r1].abs() @ hk.abs().T
        return (Stc - S).abs() + (tc_acc_steps(D) * 2.0 ** -23 + REF) * mag

    inv_T = float(np.float32(1.0 / T))
    r = nce_reference(q, k, inv_T, "tc", X.nce_geometry(n, _sms()), inv_T_ref=1.0 / T, eps=eps)
    lo = float(lo.detach())
    assert abs(r["loss"] - lo) < 1e-12
    el = abs(float(l.detach()) - lo)
    assert el <= r["E_loss"], (float(l), float(lo), r["E_loss"])
    case = "production"
    _note(("production", "loss"), case, float(l.detach()), lo, r["E_loss"])
    # F0 rows: dq at q_rows (unique), zero elsewhere
    g0, g0o = f0.grad.cpu().double(), f0o.grad.detach()
    assert not bool(np.delete(g0.numpy(), q_rows.numpy(), 0).any())
    e0 = r["E_dq"].cpu()
    assert bool(((g0[q_rows] - g0o[q_rows]).abs() <= e0).all())
    _note(("production", "dq"), case, g0[q_rows], g0o[q_rows], e0)
    # F1 rows: the dk of every key row that gathered it, summed in fp32 by the indexing backward (count - 1 roundings)
    e1 = torch.zeros(N1, D, dtype=F64).index_add_(0, k_rows, r["E_dk"].cpu())
    mag = torch.zeros(N1, D, dtype=F64).index_add_(0, k_rows, r["dk"].abs().cpu() + r["E_dk"].cpu())
    cnt = torch.zeros(N1, dtype=F64).index_add_(0, k_rows, torch.ones(n, dtype=F64))[:, None]
    e1 = e1 + (cnt - 1).clamp_min(0) * U / (1 - cnt * U) * mag
    g1, g1o = f1.grad.cpu().double(), f1o.grad.detach()
    assert bool(((g1 - g1o).abs() <= e1).all())
    used = cnt[:, 0] > 0
    _note(("production", "dk"), case, g1[used], g1o[used], e1[used])


# ----------------------------------------------------------------------------------------------- pdist_rowmin
def check_pdist(P, S, D, sms):
    """Bit-exact minval, smallest tied argmin; returns which tie geometries the case reached."""
    from pointcontrast_b200 import losses
    _, splits, sps = X.pdist_geometry(P, S, sms)
    A, B = X.pdist_operands(P, S, D, sps, seed=P * 7919 + S * 31 + D)
    mv, am = losses.pdist_rowmin(A.cuda(), B.cuda())
    Ad, Bd = A.cuda().double(), B.cuda().double()
    d2 = (Ad * Ad).sum(1)[:, None] + (Bd * Bd).sum(1)[None] - 2 * Ad @ Bd.T          # exact: multiples of 2^-12 below 4
    dmin = d2.min(1).values
    tie = d2 == dmin[:, None]
    j = torch.arange(S, device="cuda")
    jmin = torch.where(tie, j, S).min(1).values
    want = np.sqrt(dmin.cpu().numpy().astype(np.float32) + np.float32(1e-7)).astype(np.float32)
    assert np.array_equal(mv.cpu().numpy().view(np.uint32), want.view(np.uint32)), (P, S, D)
    assert torch.equal(am.long(), jmin), (P, S, D, torch.nonzero(am.long() != jmin)[:4].flatten().tolist())
    other = tie & (j != jmin[:, None])
    same_split = (j // sps)[None] == (jmin // sps)[:, None]
    same_tile = (j // X.PD_TILE)[None] == (jmin // X.PD_TILE)[:, None]
    return {name for name, m in (("same tile", other & same_tile), ("later tile", other & same_split & ~same_tile),
                                 ("other split", other & ~same_split)) if bool(m.any())}


@pytest.mark.parametrize("S", X.PD_S)
@pytest.mark.parametrize("P", X.PD_P)
def test_pdist_rowmin_bit_exact_with_smallest_tied_index(P, S):
    sms = _sms()
    _, splits, sps = X.pdist_geometry(P, S, sms)
    for D in X.PD_D:
        seen = check_pdist(P, S, D, sms)
        want = {"same tile"} if S >= 5 else set()
        want |= {"later tile"} if sps > X.PD_TILE and S > X.PD_TILE else set()
        want |= {"other split"} if splits > 1 else set()
        assert seen >= want, (P, S, D, seen, want)
