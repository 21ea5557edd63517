"""Multi-GPU plumbing for the two paths that shard (SURVEY.md section 8e): one process per
GPU, ``torch.distributed`` (NCCL over NVLink on the GPU box, gloo in the CPU tests).

* prediction over a large batch: queries are split across ranks, the model is replicated,
  there is NO data-path collective (outputs are gathered only if the caller wants them on
  every rank) -- what the reference does with ``torch.nn.DataParallel`` (predict.py:375-378);
* the K.v operator of the iterative solver: each rank evaluates a contiguous range of
  training points, then ONE all-gather of 3N*M/G doubles per iteration (iterative.py:183-204
  is the single-process operator);
* model hand-over after training on rank 0: ONE broadcast of alphas_F (+ c, std).

The compute callables are injected, so the same code runs against the CUDA engine (NCCL) and,
in the CPU tests, against the oracle (gloo).
"""

import numpy as np


def _dist():
    import torch.distributed as dist

    return dist


def world_info(group=None):
    dist = _dist()
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


def shard_bounds(n, world, rank):
    """Contiguous balanced shard [lo, hi) of range(n): the first n % world ranks get one extra."""
    base, extra = divmod(int(n), int(world))
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def _device_for_backend(group=None):
    import torch

    dist = _dist()
    backend = dist.get_backend(group)
    return torch.device('cuda', torch.cuda.current_device()) if backend == 'nccl' else torch.device('cpu')


def all_reduce_min_scalar(value, group=None):
    """min over the ranks of a host scalar (a memory budget every rank must agree on)."""
    import torch

    dist = _dist()
    if world_info(group)[1] == 1:
        return value
    t = torch.tensor([float(value)], dtype=torch.float64, device=_device_for_backend(group))
    dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
    return float(t.item())


def all_gather_rows(local, n_total, group=None):
    """Gathers row-sharded arrays (shards as produced by shard_bounds) into the full array on
    every rank.  One all_gather; shards are padded to the largest shard.  A torch tensor stays a tensor
    on its device (CUDA tensors never touch the host: NCCL moves them over NVLink); a NumPy array comes
    back as a NumPy array."""
    import torch

    dist = _dist()
    rank, world = world_info(group)
    is_tensor = hasattr(local, 'data_ptr')
    if not is_tensor:
        local = np.ascontiguousarray(local, dtype=np.float64)
    if world == 1:
        return local
    dev = _device_for_backend(group)
    loc_t = (local if is_tensor else torch.from_numpy(local)).to(dev)
    tail = tuple(loc_t.shape[1:])
    max_rows = shard_bounds(n_total, world, 0)[1]
    if n_total % world == 0:  # equal shards: gather straight into the result
        full = torch.empty((n_total,) + tail, dtype=torch.float64, device=dev)
        dist.all_gather_into_tensor(full, loc_t.contiguous(), group=group)
    else:
        buf = torch.zeros((max_rows,) + tail, dtype=torch.float64, device=dev)
        buf[: loc_t.shape[0]] = loc_t
        # gathered along the first dimension of a flat (world * max_rows) tensor: gloo takes no stacked output
        out = torch.empty((world * max_rows,) + tail, dtype=torch.float64, device=dev)
        dist.all_gather_into_tensor(out, buf, group=group)
        out = out.view((world, max_rows) + tail)
        full = torch.cat([out[r, : shard_bounds(n_total, world, r)[1] - shard_bounds(n_total, world, r)[0]] for r in range(world)], dim=0)
    if is_tensor:
        return full.to(local.device)
    return full.cpu().numpy()


def exchange_on_workspace(ws, off, count, op, n_train, dim_i, group=None):
    """The exchange function of `sgdml_b200_pcg` (include/sgdml_b200.h) on torch.distributed: `ws` is the
    solver's device workspace (a flat float64 tensor), [off, off + count) the buffer of this exchange.
      op 0: sum over the ranks in place (X^T v of the row-sharded Nystroem factor, m doubles);
      op 1: all-gather of a replicated n-vector whose rows [lo*dim_i, hi*dim_i) this rank has just written
            (K.v rows, P.v rows): in place when the shards are equal, through a padded staging tensor otherwise;
      op 2: the same for the M-entry energy tail of an energy-constrained solve (sgdml_b200_pcg_ecstr): entries
            [lo, hi) are this rank's.
    Collectives are enqueued in stream order on the backend's stream; nothing is copied to the host."""
    import torch

    dist = _dist()
    rank, world = world_info(group)
    view = ws[off : off + count]
    if world == 1:
        return
    if op == 0:
        dist.all_reduce(view, op=dist.ReduceOp.SUM, group=group)
        return
    if op not in (1, 2):
        raise ValueError('unknown exchange op %r' % (op,))
    if op == 2:
        dim_i = 1  # one energy entry per training point
    assert count == n_train * dim_i
    lo, hi = shard_bounds(n_train, world, rank)
    if n_train % world == 0:
        dist.all_gather_into_tensor(view, view[lo * dim_i : hi * dim_i], group=group)
        return
    max_rows = shard_bounds(n_train, world, 0)[1] * dim_i
    buf = torch.zeros(max_rows, dtype=ws.dtype, device=ws.device)
    buf[: (hi - lo) * dim_i] = view[lo * dim_i : hi * dim_i]
    out = torch.empty(world * max_rows, dtype=ws.dtype, device=ws.device)
    dist.all_gather_into_tensor(out, buf, group=group)
    for r in range(world):
        rlo, rhi = shard_bounds(n_train, world, r)
        if r != rank:
            view[rlo * dim_i : rhi * dim_i] = out[r * max_rows : r * max_rows + (rhi - rlo) * dim_i]


def predict_sharded(predict_fn, R, gather=True, group=None):
    """predict_fn(R_shard) -> (E, F).  Splits the query batch across ranks; with gather=True every
    rank receives the full (E, F), otherwise each rank keeps (lo, hi, E_local, F_local)."""
    rank, world = world_info(group)
    R = np.asarray(R, dtype=np.float64)
    n = R.shape[0]
    lo, hi = shard_bounds(n, world, rank)
    E, F = predict_fn(R[lo:hi])
    if not gather:
        return lo, hi, E, F
    return all_gather_rows(E, n, group), all_gather_rows(F, n, group)


def predict_virial_sharded(predict_virial_fn, R, lattice=None, gather=True, group=None):
    """predict_virial_fn(R_shard, lattice_shard) -> (E, F, W) (GDMLPredict.predict_virial).  Splits the query batch
    across ranks like `predict_sharded`; a (B, 3, 3) `lattice` (one cell per geometry) is split with it, a (3, 3) one or
    None goes to every rank as it is.  With gather=True every rank receives the full (E, F, W), otherwise each rank
    keeps (lo, hi, E_local, F_local, W_local)."""
    rank, world = world_info(group)
    R = np.asarray(R, dtype=np.float64)
    n = R.shape[0]
    lo, hi = shard_bounds(n, world, rank)
    lat = None
    if lattice is not None:
        if hasattr(lattice, 'data_ptr'):
            lattice = lattice.detach().cpu().numpy()
        lat = np.asarray(lattice, dtype=np.float64)
        if lat.ndim == 3:
            if lat.shape[0] != n:
                raise ValueError('lattice holds %d cells for %d geometries' % (lat.shape[0], n))
            lat = lat[lo:hi]
    E, F, W = predict_virial_fn(R[lo:hi], lat)
    if not gather:
        return lo, hi, E, F, W
    return all_gather_rows(E, n, group), all_gather_rows(F, n, group), all_gather_rows(W, n, group)


def kmatvec_sharded(rows_fn, n_train, group=None):
    """rows_fn(m_lo, m_hi) -> (m_hi - m_lo, 3N) raw force sums for training points [m_lo, m_hi)
    (GDMLPredict.kmatvec_train).  Returns the full (n_train, 3N) product on every rank after one
    all-gather."""
    rank, world = world_info(group)
    lo, hi = shard_bounds(n_train, world, rank)
    return all_gather_rows(rows_fn(lo, hi), n_train, group)


def broadcast_coefficients(alphas_F, c, std, src=0, group=None):
    """One broadcast of [alphas_F, c, std] from `src`; returns (alphas_F, c, std) on every rank.
    On ranks != src, `alphas_F` only needs the right length."""
    import torch

    dist = _dist()
    rank, world = world_info(group)
    a = np.ascontiguousarray(alphas_F, dtype=np.float64)
    if world == 1:
        return a, float(c), float(std)
    dev = _device_for_backend(group)
    buf = torch.empty(a.size + 2, dtype=torch.float64, device=dev)
    if rank == src:
        buf[: a.size] = torch.from_numpy(a).to(dev)
        buf[a.size] = float(c)
        buf[a.size + 1] = float(std)
    dist.broadcast(buf, src=src, group=group)
    host = buf.cpu().numpy()
    return host[: a.size].copy(), float(host[a.size]), float(host[a.size + 1])


# --------------------------------------------------------------------------- row-sharded Nystroem factor
# SURVEY.md section 8e, rows "explicit K assembly" and "Nystroem factor (m, n): shard n": each rank
# assembles and keeps only the block rows of K_nm that belong to its own training points.  The two
# small (m x m) matrices are summed over the ranks (this is the all-reduce BASELINE config 4 names),
# factorised redundantly (bit-identical on every rank), and applied to the local rows.  The
# algorithms are written as generators that yield at every exchange:
#   ('sum', tensor)      -> the tensor is summed over the ranks in place
#   ('gather', rows)     -> the row-sharded NumPy array is gathered; the full array is sent back
# `run_steps` drives one generator with torch.distributed; `run_steps_virtual` drives the generators
# of several virtual ranks in lockstep inside ONE process (single-GPU tests of the sharded path).
# `ops` supplies the compute (the CUDA engine in solvers/iterative.py; NumPy stand-ins in the CPU tests).


def all_reduce_sum_(t, group=None):
    """In-place sum over the ranks of a torch tensor living on the backend's device."""
    dist = _dist()
    if world_info(group)[1] > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


def _own_rows(cols, lo, hi, n_train, dim_i, use_E_cstr):
    """Positions in `cols` of the inducing columns whose rows live on the rank with training points [lo, hi), and
    their rows in that rank's block.  With energy constraints the block is the force rows of [lo, hi), then their
    energy rows, and energy column c >= 3NM belongs to point c - 3NM."""
    n_f = n_train * dim_i
    own = np.nonzero((cols >= lo * dim_i) & (cols < hi * dim_i))[0]
    local = cols[own] - lo * dim_i
    if use_E_cstr:
        own_e = np.nonzero((cols >= n_f + lo) & (cols < n_f + hi))[0]
        own = np.concatenate([own, own_e])
        local = np.concatenate([local, (hi - lo) * dim_i + (cols[own_e] - n_f - lo)])
    return own, local


def nystroem_factor_steps(ops, rank, world, n_train, dim_i, cols, lam, use_E_cstr=False):
    """Row-sharded iterative.py:208-351.  Returns (X_loc, lo, hi): the rows [lo*dim_i, hi*dim_i) of
    the factor B^T = K_nm L^-T L_inner^-T (first len(cols) columns of X_loc).  use_E_cstr: the system is
    (3NM + M)-square, `cols` index its columns, and X_loc holds the force rows of [lo, hi), then their energy
    rows (ops.assemble_rows returns that block)."""
    lo, hi = shard_bounds(n_train, world, rank)
    cols = np.ascontiguousarray(cols, dtype=np.int64)
    m = len(cols)
    X = ops.assemble_rows(lo, hi, cols)  # local rows of K_nm (iterative.py:237-247)
    own, local = _own_rows(cols, lo, hi, n_train, dim_i, use_E_cstr)
    A = ops.new_square(m)
    ops.put_neg_rows(A, own, X, local, m)  # rows of K_mm = -K_nm[cols] owned here (iterative.py:253)
    yield 'sum', A
    if not ops.cho_factor_stable(A, pre_reg=True):  # iterative.py:267
        raise np.linalg.LinAlgError('Failed to factorize K_mm despite strong regularization')
    ops.trsm_right_lt(A, X, m)  # iterative.py:278-287 on the local rows
    ops.gram(X, m, A)  # local part of K_nm^T K_nm (iterative.py:293-295)
    yield 'sum', A
    ops.add_diag(A, m, lam)
    if ops.cho_factor_stable(A, eps_mag_max=-14):  # do not regularize more than 1e-14 (iterative.py:305-307)
        ops.trsm_right_lt(A, X, m)  # iterative.py:337-347
    else:
        # iterative.py:312-322: the reference takes the R factor of a Householder QR of the stacked
        # ((n + m) x m) matrix [K_nm; sqrt(lam) I] and solves with it.  R^T R is the same inner matrix,
        # so X R^-1 is the top block of the thin Q factor; it is formed here by shifted CholeskyQR3
        # (three Gram + Cholesky + triangular-solve passes, the first one shifted), which is
        # backward stable for condition numbers up to ~1/eps and needs only the (m x m) all-reduce.
        n_rows = n_train * dim_i + (n_train if use_E_cstr else 0)
        Y = ops.scaled_identity(m, np.sqrt(lam))  # the bottom block, replicated on every rank
        for it in range(3):
            ops.gram(X, m, A)
            yield 'sum', A
            ops.add_gram(Y, m, A)
            if it == 0:
                eps = np.finfo(float).eps
                ops.add_diag(A, m, 11.0 * (m * (n_rows + m) + m * (m + 1)) * eps * ops.trace(A, m))
            if not ops.potrf(A):
                raise np.linalg.LinAlgError('QR fallback of the Nystroem factor failed (matrix not positive definite)')
            ops.trsm_right_lt(A, X, m)
            ops.trsm_right_lt(A, Y, m)
    return X, lo, hi


def lev_scores_steps(ops, X, m, dim_i, use_E_cstr=False):
    """Leverage scores (iterative.py:107-109) of a row-sharded factor, gathered on every rank.  use_E_cstr: the
    force part and the energy part of the local rows are gathered separately, into [forces; energies]."""
    sq = ops.row_sqnorms(X, m)
    if not use_E_cstr:
        full = yield 'gather', sq.reshape(-1, dim_i)
        return full.ravel()
    n_f_loc = sq.size // (dim_i + 1) * dim_i
    full_f = yield 'gather', sq[:n_f_loc].reshape(-1, dim_i)
    full_e = yield 'gather', sq[n_f_loc:].reshape(-1, 1)
    return np.concatenate([np.asarray(full_f).ravel(), np.asarray(full_e).ravel()])


def precon_apply_steps(ops, X, m, lam, v, lo, hi, dim_i, use_E_cstr=False):
    """P v = (B^T (B v) - v)/lam (iterative.py:136-138) with B^T row-sharded: one m-vector
    all-reduce and one all-gather of the n-vector per application (two with use_E_cstr: the force part and the
    energy tail of v = [forces; energies])."""
    v_loc = np.ascontiguousarray(v[lo * dim_i : hi * dim_i], dtype=np.float64)
    if use_E_cstr:
        n_f = len(v) // (dim_i + 1) * dim_i
        v_loc = np.concatenate([v_loc, np.asarray(v[n_f + lo : n_f + hi], dtype=np.float64)])
    t = ops.project(X, m, v_loc)
    yield 'sum', t
    out_loc = ops.expand(X, m, lam, t, v_loc)
    if not use_E_cstr:
        full = yield 'gather', out_loc.reshape(-1, dim_i)
        return full.ravel()
    n_f_loc = (hi - lo) * dim_i
    full_f = yield 'gather', out_loc[:n_f_loc].reshape(-1, dim_i)
    full_e = yield 'gather', out_loc[n_f_loc:].reshape(-1, 1)
    return np.concatenate([np.asarray(full_f).ravel(), np.asarray(full_e).ravel()])


def run_steps(gen, n_train, group=None):
    """Drives one rank's generator with torch.distributed collectives."""
    try:
        op, payload = next(gen)
        while True:
            if op == 'sum':
                all_reduce_sum_(payload, group)
                res = None
            elif op == 'gather':
                res = all_gather_rows(payload, n_train, group)
            else:
                raise ValueError(op)
            op, payload = gen.send(res)
    except StopIteration as e:
        return e.value


def run_steps_virtual(gens):
    """Drives the generators of len(gens) virtual ranks in lockstep in this process; returns their
    return values.  Same exchanges as run_steps, done by hand."""
    world = len(gens)
    results = [None] * world
    msgs = [next(g) for g in gens]
    while True:
        ops_ = {op for op, _ in msgs}
        assert len(ops_) == 1, 'virtual ranks diverged'
        op = ops_.pop()
        if op == 'sum':
            total = msgs[0][1].clone()
            for _, t in msgs[1:]:
                total += t
            for _, t in msgs:
                t.copy_(total)
            sends = [None] * world
        elif op == 'gather':
            full = np.concatenate([np.asarray(p) for _, p in msgs], axis=0)
            sends = [full] * world
        else:
            raise ValueError(op)
        nxt, done = [], 0
        for r, g in enumerate(gens):
            try:
                nxt.append(g.send(sends[r]))
            except StopIteration as e:
                results[r] = e.value
                done += 1
        if done == world:
            return results
        assert done == 0, 'virtual ranks diverged'
        msgs = nxt


# --------------------------------------------------------------------------- prediction sharded over training points
def model_shard(model, lo, hi):
    """The part of a model dict that belongs to training points [lo, hi), as a raw-sum model
    (std = 1, c = 0): predictions of the shards add up to the unscaled prediction of `model`."""
    n_train = model['R_desc'].shape[1]
    sub = dict(model)
    sub['R_desc'] = np.ascontiguousarray(np.asarray(model['R_desc'])[:, lo:hi])  # stored (D, M), train.py:807
    sub['R_d_desc_alpha'] = np.ascontiguousarray(np.asarray(model['R_d_desc_alpha'])[lo:hi])
    sub['alphas_F'] = np.asarray(model['alphas_F']).reshape(n_train, -1)[lo:hi].ravel()
    if 'alphas_E' in model:  # energy-constrained models: one coefficient per training point
        sub['alphas_E'] = np.asarray(model['alphas_E']).ravel()[lo:hi]
    if 'idxs_train' in model:
        sub['idxs_train'] = np.asarray(model['idxs_train'])[lo:hi]
    sub['std'] = 1.0
    sub['c'] = 0.0
    return sub


class TrainPointShardedPredictor(object):
    """SURVEY.md section 8e "predict, small B / huge M*S": the sum over training points is split
    across the ranks (M/G points each, predict.py:1280-1284 already sums partial results), every
    rank evaluates the WHOLE query batch against its shard, then ONE all-reduce of B*(3N+1) doubles
    (the back-projection J^T is linear, so the partial forces are summed after it).

    predictor_cls(model) must offer .predict(R) -> (E, F), and .predict_virial(R, lattice=...) -> (E, F, W) for
    `predict_virial`: sgdml_b200.GDMLPredict on the GPU box, the oracle predictor in the CPU tests."""

    def __init__(self, model, predictor_cls, group=None):
        self.group = group
        rank, world = world_info(group)
        n_train = model['R_desc'].shape[1]
        self.lo, self.hi = shard_bounds(n_train, world, rank)
        self.std = float(model['std']) if 'std' in model else 1.0
        self.c = float(model['c'])
        self.dim_i = 3 * int(np.asarray(model['z']).shape[0])
        self.part = predictor_cls(model_shard(model, self.lo, self.hi)) if self.hi > self.lo else None

    def predict(self, R, return_E=True):
        """R: NumPy array (B, 3N) -> NumPy (E, F); or a CUDA float64 tensor -> CUDA tensors, in which case the
        partial results, the all-reduce (NCCL) and the scaling all stay on the device."""
        import torch

        on_device = hasattr(R, 'data_ptr') and R.is_cuda
        if not on_device:
            R = np.asarray(R, dtype=np.float64)
            if R.ndim == 1:
                R = R[None, :]  # predict.py:1183-1184
            B = R.shape[0]
            buf = np.zeros((B, self.dim_i + 1))
            if self.part is not None:
                E, F = self.part.predict(R)
                buf[:, 0], buf[:, 1:] = E, F.reshape(B, -1)
            if world_info(self.group)[1] > 1:
                t = torch.from_numpy(buf).to(_device_for_backend(self.group))
                all_reduce_sum_(t, self.group)
                buf = t.cpu().numpy()
            F = buf[:, 1:] * self.std  # predict.py:1286-1288
            if not return_E:
                return (F,)
            return buf[:, 0] * self.std + self.c, F
        R = R.reshape(-1, self.dim_i)
        B = R.shape[0]
        # one buffer [F | E] so that ONE all-reduce of B*(3N+1) doubles carries both (SURVEY 8e)
        buf = torch.zeros(B * (self.dim_i + 1), dtype=torch.float64, device=R.device)
        F_v = buf[: B * self.dim_i].view(B, self.dim_i)
        E_v = buf[B * self.dim_i :]
        if self.part is not None:
            self.part.predict(R, out=(E_v, F_v))
        all_reduce_sum_(buf, self.group)
        F_v *= self.std
        if not return_E:
            return (F_v,)
        E_v *= self.std
        E_v += self.c
        return E_v, F_v

    def predict_virial(self, R, lattice=None, return_E=True):
        """`predict` plus the virial: R and lattice as GDMLPredict.predict_virial ((3, 3), one cell per geometry
        (B, 3, 3), or None for the model's own) -> (E, F, W) or (F, W).  W is linear in F_desc, hence in the sum over
        training points, so each rank's raw shard virial (std = 1, c = 0) rides in the same ONE all-reduce as E and F:
        a buffer [F | E | W] of B*(3N+10) doubles.  std and c are applied afterwards.  CUDA tensors stay on the device
        (NCCL)."""
        import torch

        on_device = hasattr(R, 'data_ptr') and R.is_cuda
        if on_device:
            R = R.reshape(-1, self.dim_i)
            B = R.shape[0]
            buf = torch.zeros(B * (self.dim_i + 10), dtype=torch.float64, device=R.device)
        else:
            R = np.asarray(R, dtype=np.float64).reshape(-1, self.dim_i)
            B = R.shape[0]
            buf = torch.zeros(B * (self.dim_i + 10), dtype=torch.float64)
        F_v = buf[: B * self.dim_i].view(B, self.dim_i)
        E_v = buf[B * self.dim_i : B * (self.dim_i + 1)]
        W_v = buf[B * (self.dim_i + 1) :].view(B, 3, 3)
        if self.part is not None:
            if on_device:
                self.part.predict_virial(R, lattice=lattice, out=(E_v, F_v, W_v))
            else:
                E, F, W = self.part.predict_virial(R, lattice=lattice)
                E_v.copy_(torch.from_numpy(np.asarray(E, dtype=np.float64)))
                F_v.copy_(torch.from_numpy(np.asarray(F, dtype=np.float64).reshape(B, -1)))
                W_v.copy_(torch.from_numpy(np.asarray(W, dtype=np.float64).reshape(B, 3, 3)))
        if world_info(self.group)[1] > 1:
            if on_device:
                all_reduce_sum_(buf, self.group)
            else:
                t = buf.to(_device_for_backend(self.group))
                all_reduce_sum_(t, self.group)
                buf.copy_(t.cpu())
        F_v *= self.std
        W_v *= self.std
        E_v *= self.std
        E_v += self.c
        if not on_device:
            F_v, E_v, W_v = F_v.numpy(), E_v.numpy(), W_v.numpy()
        return (E_v, F_v, W_v) if return_E else (F_v, W_v)
