"""Host-side mirror of the parts of the reference's ``utils.py`` / ``visualization.py`` that sit on the
compression-matrix path of SaveCompressionMatricesCallback (SURVEY.md section 8 a14)."""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import _lib


def _dev(a, device):
    t = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))
    return t.to(device=device, dtype=torch.float32).contiguous()


def _pairwise(kind, mus1, logvars1, mus2, logvars2, device):
    if not torch.cuda.is_available():
        raise _lib.DibError("dib_b200 needs a CUDA device; there is no CPU path")
    lib = _lib.load()
    device = device or (mus1.device if isinstance(mus1, torch.Tensor) and mus1.is_cuda
                        else torch.device("cuda", torch.cuda.current_device()))
    ml1 = torch.cat([_dev(mus1, device), _dev(logvars1, device)], dim=1).contiguous()
    same = mus2 is None or (mus2 is mus1 and logvars2 is logvars1)
    ml2 = ml1 if same else torch.cat([_dev(mus2, device), _dev(logvars2, device)], dim=1).contiguous()
    if ml1.shape[1] != ml2.shape[1]:
        raise ValueError("embedding dimensions differ")
    n, m, E = ml1.shape[0], ml2.shape[0], ml1.shape[1] // 2
    out = torch.empty(n, m, dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        _lib.check(lib.dib_pairwise_gaussian(kind, _lib.ptr(ml1), n, _lib.ptr(ml2), m, E, _lib.ptr(out), None,
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out if isinstance(mus1, torch.Tensor) else out.cpu().numpy()


def bhattacharyya_dist_mat(mus1, logvars1, mus2=None, logvars2=None, device=None):
    """utils.py:177-212 (Bhattacharyya distances between diagonal Gaussians, [N, M]) on the GPU in the O(N*M*E)
    closed form (dib_pairwise_gaussian kind 0)."""
    return _pairwise(0, mus1, logvars1, mus2, logvars2, device)


def kl_divergence_mat(mus1, logvars1, mus2=None, logvars2=None, device=None):
    """utils.py:213-247: KL(N(mus1_i, e^logvars1_i) || N(mus2_j, e^logvars2_j)), [N, M] (dib_pairwise_gaussian kind 1)."""
    return _pairwise(1, mus1, logvars1, mus2, logvars2, device)


def select_display_rows(inp_features_raw, max_number_to_display=128, rng=None):
    """visualization.py:17-28: unique values if fewer than 10 distinct, else ``max_number_to_display`` random rows,
    sorted by raw value.  Returns (row indices into the input, sorted raw values)."""
    raw = np.asarray(inp_features_raw)
    flat = raw.reshape(raw.shape[0], -1)[:, 0]
    unique_vals, unique_inds = np.unique(flat, return_index=True)
    if len(unique_vals) < 10:
        return unique_inds[np.argsort(unique_vals)], np.sort(unique_vals)
    rng = rng or np.random.default_rng()
    sel = rng.choice(flat.shape[0], max_number_to_display)
    order = np.argsort(flat[sel])
    return sel[order], flat[sel][order]


def compression_matrix(feature_encoder, feature_inps):
    """visualization.py:30-34: encoder forward -> (mu, logvar) -> Bhattacharyya -> exp(-D).
    Returns (compression_matrix, bhattacharyya_distance_matrix) as numpy arrays."""
    lib = _lib.load()
    model = feature_encoder._model
    o = model._encode_feature(feature_encoder.index, feature_inps)            # [n, 2E] on the device
    n, E = o.shape[0], model.feature_embedding_dimension
    dist = torch.empty(n, n, dtype=torch.float32, device=o.device)
    comp = torch.empty(n, n, dtype=torch.float32, device=o.device)
    with torch.cuda.device(o.device):
        _lib.check(lib.dib_bhattacharyya(_lib.ptr(o), n, E, _lib.ptr(dist), _lib.ptr(comp),
                                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return comp.cpu().numpy(), dist.cpu().numpy()


def mi_sandwich_batch(mu_logvar, eps=None, seed=0, step=0):
    """One batch of utils.py:36-65 on the GPU (dib_mi_sandwich_bounds): (InfoNCE lower, leave-one-out upper) in nats.
    ``mu_logvar`` [n, 2E] on the device; ``eps`` [n, E] or None (Philox)."""
    lib = _lib.load()
    n, E = mu_logvar.shape[0], mu_logvar.shape[1] // 2
    dev = mu_logvar.device
    scratch = torch.empty(2 * n, dtype=torch.float32, device=dev)
    out = torch.empty(2, dtype=torch.float32, device=dev)
    e = None if eps is None else _dev(eps, dev)
    with torch.cuda.device(dev):
        _lib.check(lib.dib_mi_sandwich_bounds(_lib.ptr(mu_logvar.contiguous()), n, E, _lib.ptr(e), int(seed), int(step) & 0xFFFFFFFF,
                                              _lib.ptr(scratch), _lib.ptr(out),
                                              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out


def estimate_mi_sandwich_bounds(encoder, dataset, evaluation_batch_size=1024, number_evaluation_batches=8, seed=0):
    """utils.py:10-73: upper and lower bounds of the information transmitted by one feature encoder.

    ``encoder`` is ``model.feature_encoders[i]``; ``dataset`` the rows of that feature ([N, d_i] array or tensor; a
    ``(x, y)`` tuple is accepted and y dropped, as the reference's callback does).  Batches are drawn like the
    reference's ``repeat().shuffle().batch().take()``: ``number_evaluation_batches`` batches of
    ``evaluation_batch_size`` rows sampled (with our seeded RNG; the reference's shuffle is unseeded) from the
    repeated data.  Returns np.array([lower, upper]) in nats, the mean over batches."""
    if isinstance(dataset, (tuple, list)):
        dataset = dataset[0]
    model = encoder._model
    x = _dev(dataset, model.device)
    if x.dim() == 1:
        x = x[:, None]
    N = x.shape[0]
    gen = torch.Generator(device=model.device)
    gen.manual_seed(int(seed))
    outs = []
    for b in range(int(number_evaluation_batches)):
        idx = torch.randint(0, N, (int(evaluation_batch_size),), generator=gen, device=model.device)
        o = model._encode_feature(encoder.index, x.index_select(0, idx))
        outs.append(mi_sandwich_batch(o, None, seed=(int(seed) << 8) + encoder.index, step=b))
    return torch.stack(outs).mean(0).double().cpu().numpy()


def estimate_mi_sandwich_bounds_all_features(model, x, evaluation_batch_size=1024, number_evaluation_batches=8, seed=0):
    """utils.py:10-73 for EVERY feature encoder of ``model`` at once (what InfoPerFeatureCallback, models.py:188-223, loops
    over in Python): one grouped encoder forward on the gathered rows (dib_compression_matrices) and ONE launch of the
    batched float64 sandwich kernel (dib_mi_sandwich_bounds_batched) over features x batches groups.  Row draws and noise
    streams are those of the per-feature ``estimate_mi_sandwich_bounds`` calls with the same ``seed``.
    ``x``: [N, sum d_i] rows (a ``(x, y)`` tuple is accepted).  Returns a float64 array [F, 2] = (lower, upper) in nats."""
    if isinstance(x, (tuple, list)):
        x = x[0]
    lib = _lib.load()
    xd = _dev(x, model.device)
    N, F, E = xd.shape[0], model.number_features, model.feature_embedding_dimension
    bs, nb = int(evaluation_batch_size), int(number_evaluation_batches)
    gen = torch.Generator(device=model.device)
    gen.manual_seed(int(seed))
    idx = torch.cat([torch.randint(0, N, (bs,), generator=gen, device=model.device) for _ in range(nb)])
    row_index = idx.to(torch.int32).unsqueeze(0).expand(F, -1).contiguous()
    ml = model.compression_matrices(xd, row_index, want=("mu_logvar",))["mu_logvar"]          # [F, nb * bs, 2E]
    scratch = torch.empty(F * nb * bs * 2, dtype=torch.float64, device=model.device)
    out = torch.empty(F * nb, 2, dtype=torch.float64, device=model.device)
    with torch.cuda.device(model.device):
        _lib.check(lib.dib_mi_sandwich_bounds_batched(_lib.ptr(ml), F * nb, bs, E, None, int(seed), nb, _lib.ptr(scratch),
                                                      _lib.ptr(out), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out.view(F, nb, 2).mean(1).cpu().numpy()


def mi_bounds_at_probes(probe_mu_logvar, data_mu_logvar, batch_offsets, eps=None, seed=0):
    """nb-particle cell 8 (:549-570) on the GPU (dib_mi_bounds_at_probes): per-probe (InfoNCE lower, leave-one-out upper)
    bounds in nats, float64 [M, 2], of probe encodings ``probe_mu_logvar`` [M, 2E] against the batches of encoded data
    rows ``data_mu_logvar`` [R, 2E], batch b being rows ``batch_offsets[b] .. batch_offsets[b + 1]`` (B + 1 nondecreasing
    int64 offsets, every batch at least one row).  ``eps`` [B, M, E] or None (Philox keyed by seed, batch and probe)."""
    lib = _lib.load()
    dev = data_mu_logvar.device
    P = probe_mu_logvar.to(device=dev, dtype=torch.float32).contiguous()
    D = data_mu_logvar.to(dtype=torch.float32).contiguous()
    if P.dim() != 2 or D.dim() != 2 or P.shape[1] != D.shape[1] or P.shape[1] % 2:
        raise ValueError(f"probe and data encodings must be [rows, 2E] of one E, got {tuple(P.shape)} and {tuple(D.shape)}")
    M, R, E = P.shape[0], D.shape[0], P.shape[1] // 2
    if not (isinstance(batch_offsets, torch.Tensor) and batch_offsets.is_cuda):
        o = np.asarray(batch_offsets.cpu() if isinstance(batch_offsets, torch.Tensor) else batch_offsets, dtype=np.int64)
        if o.ndim != 1 or o.size < 2 or o[0] < 0 or o[-1] > R or np.any(np.diff(o) < 1):
            raise ValueError("batch_offsets must be B + 1 increasing offsets in [0, rows]: every batch needs a row")
    off = torch.as_tensor(batch_offsets).to(device=dev, dtype=torch.int64).contiguous()
    B = off.numel() - 1
    e = None
    if eps is not None:
        e = _dev(eps, dev)
        if tuple(e.shape) != (B, M, E):
            raise ValueError(f"eps has shape {tuple(e.shape)}; expected {(B, M, E)}")
    scratch = torch.empty(int(lib.dib_mi_bounds_at_probes_scratch_bytes(M, R, B, E)), dtype=torch.uint8, device=dev)
    out = torch.empty(M, 2, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.dib_mi_bounds_at_probes(_lib.ptr(P), M, _lib.ptr(D), _lib.ptr(off), B, E, _lib.ptr(e), int(seed),
                                               _lib.ptr(scratch), _lib.ptr(out),
                                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out


def draw_evaluation_batches(number_items, evaluation_batch_size, number_evaluation_batches, seed, device):
    """The evaluation draws of :func:`estimate_mi_bounds_at_probes` and :func:`estimate_set_information`: a
    ``torch.Generator(device)`` seeded with ``seed``, then for b = 0, 1, ... in order
    ``torch.randint(0, number_items, (evaluation_batch_size,), generator=gen, device=device)``.  Returns [B, bs] int64."""
    gen = torch.Generator(device=device)
    gen.manual_seed(int(seed))
    return torch.stack([torch.randint(0, int(number_items), (int(evaluation_batch_size),), generator=gen, device=device)
                        for _ in range(int(number_evaluation_batches))])


def set_batch_rows(set_index, set_sizes, set_length):
    """Particle rows of drawn sets: ``set_index`` [B, bs] set numbers, ``set_sizes`` [N] real particles per set (None: all
    ``set_length``).  Returns (rows, offsets): the indices into the [N * set_length] particle rows of every real particle,
    batch by batch, set by set, particle by particle, and the B + 1 batch offsets into ``rows``.  Works on any device."""
    L = int(set_length)
    idx = set_index.to(torch.int64)
    ar = torch.arange(L, device=idx.device)
    if set_sizes is None:
        sz = torch.full_like(idx, L)
    else:
        sz = torch.as_tensor(set_sizes).to(device=idx.device, dtype=torch.int64)[idx]
    rows = (idx[..., None] * L + ar)[ar < sz[..., None]]
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64, device=idx.device), torch.cumsum(sz.sum(1), 0)])
    return rows, offsets


def _particle_sets(model, dataset):
    """Sets for a SetTransformerIBNet: [N, L, d] (a fixed-size model also takes an (x, y) pair), or for a variable-size
    model a list of [l_i, d] or a pair (x_padded, set_sizes).  Returns (particle rows [N * L, d] on the device, set count
    N, int64 device sizes or None)."""
    from .models import pad_sets
    L, d = model.number_particles, model.particle_feature_dimensions
    sizes = None
    if model.variable_set_sizes and isinstance(dataset, list):
        dataset = pad_sets(dataset, L)
    if isinstance(dataset, tuple):
        if model.variable_set_sizes:
            dataset, sizes = dataset
        else:
            dataset = dataset[0]
    N = dataset.shape[0]
    x = model._to_device(dataset, L * d).reshape(N * L, d)
    if sizes is not None:
        sizes = model._device_sizes(sizes, N).to(torch.int64)
    return x, N, sizes


def _encode_within_handle(model, i, rows):
    """Encoder i (no noise, logvar offset applied) on ``rows`` in chunks that fit the model's handle, so that encoding
    never re-creates it (that would re-allocate the training workspace and drop the captured CUDA graphs); a model without
    a handle gets the smallest one."""
    if model._handle is None:
        model._ensure_handle(1)
    per = model._max_batch * getattr(model, "number_particles", 1)
    out = torch.empty(rows.shape[0], 2 * model.feature_embedding_dimension, dtype=torch.float32, device=model.device)
    for a in range(0, rows.shape[0], per):
        out[a:a + per] = model._encode_feature(i, rows[a:a + per])
    return out


def estimate_mi_bounds_at_probes(encoder, probes, dataset, evaluation_batch_size=512, number_evaluation_batches=16, seed=0):
    """Per-probe information map (nb-particle cell 8, :521-570): for every probe input, the InfoNCE lower and the
    leave-one-out upper bound (nats) of the information its encoding carries, against ``number_evaluation_batches``
    batches of data.  Returns float64 [M, 2] (lower, upper); the notebook plots mean(lower, upper) / ln 2.

    ``encoder`` is ``model.particle_encoder`` of a SetTransformerIBNet -- ``probes`` [M, d] particle rows, ``dataset`` sets
    ([N, L, d]; for a variable-size model also a list of [l_i, d] or a pair (x_padded, set_sizes)); a batch draws
    ``evaluation_batch_size`` sets and holds all their real particles, padding rows never enter -- or
    ``model.feature_encoders[i]`` -- ``probes`` [M, d_i], ``dataset`` rows [N, d_i] (an (x, y) pair: x); a batch draws
    ``evaluation_batch_size`` rows.  Draws: :func:`draw_evaluation_batches` (``seed``) over the sets or rows, then for sets
    :func:`set_batch_rows`.  Probes and data rows are encoded without noise (logvar offset included) within the model's
    current handle; training state (handle, graphs, step counters, noise streams) is left as it was.  The sample noise is
    Philox keyed (seed, batch, probe), so a probe's result does not depend on the other probes.

    The notebook draws fresh batches for every chunk of 100 probes; here the batches are drawn once and every probe is
    scored against them.  Each probe's estimator has the same distribution either way, only the correlation between
    probes changes, and the data rows are encoded once instead of once per chunk."""
    from .models import _ParticleEncoder
    model = encoder._model
    dev = model.device
    bs, nb = int(evaluation_batch_size), int(number_evaluation_batches)
    if isinstance(encoder, _ParticleEncoder):
        x, N, sizes = _particle_sets(model, dataset)
        rows, off = set_batch_rows(draw_evaluation_batches(N, bs, nb, seed, dev), sizes, model.number_particles)
        d = model.particle_feature_dimensions
    else:
        if isinstance(dataset, (tuple, list)):
            dataset = dataset[0]
        d = model.feature_dimensionalities[encoder.index]
        x = _dev(dataset, dev).reshape(-1, d)
        rows = draw_evaluation_batches(x.shape[0], bs, nb, seed, dev).reshape(-1)
        off = torch.arange(nb + 1, dtype=torch.int64, device=dev) * bs
    p = _dev(probes, dev).reshape(-1, d)
    data = _encode_within_handle(model, encoder.index, x.index_select(0, rows))
    ml_probes = _encode_within_handle(model, encoder.index, p)
    return mi_bounds_at_probes(ml_probes, data, off, None, seed).cpu().numpy()


def estimate_set_information(model, x, evaluation_batch_size=32, number_evaluation_batches=16, seed=0):
    """nb-particle's ``info_bounds`` (:502-517), the x-axis of its information plane: [lower, upper] in nats per set of a
    SetTransformerIBNet.  Sets are drawn with :func:`draw_evaluation_batches` (``seed``); the batch bounds of all the real
    particles of a batch come from dib_mi_sandwich_bounds_batched (float64, E <= 64) and are multiplied by the particles
    per set: number_particles, or for variable sizes the batch's mean drawn size.  Fixed sizes: one launch, batch b on the
    noise stream (seed << 8) at step b; variable sizes: one launch per batch, on stream ((seed << 16) + b) << 8."""
    lib = _lib.load()
    xr, N, sizes = _particle_sets(model, x)
    L, E = model.number_particles, model.feature_embedding_dimension
    bs, nb = int(evaluation_batch_size), int(number_evaluation_batches)
    rows, off = set_batch_rows(draw_evaluation_batches(N, bs, nb, seed, model.device), sizes, L)
    ml = _encode_within_handle(model, 0, xr.index_select(0, rows))
    stream = ctypes.c_void_p(torch.cuda.current_stream(model.device).cuda_stream)
    with torch.cuda.device(model.device):
        if sizes is None:
            n = bs * L
            scratch = torch.empty(nb * n * 2, dtype=torch.float64, device=model.device)
            out = torch.empty(nb, 2, dtype=torch.float64, device=model.device)
            _lib.check(lib.dib_mi_sandwich_bounds_batched(_lib.ptr(ml), nb, n, E, None, int(seed), nb, _lib.ptr(scratch),
                                                          _lib.ptr(out), stream))
            per_set = out * L
        else:
            oh = off.cpu().tolist()
            per_set = torch.empty(nb, 2, dtype=torch.float64, device=model.device)
            scratch = torch.empty(2 * max(b1 - b0 for b0, b1 in zip(oh[:-1], oh[1:])), dtype=torch.float64,
                                  device=model.device)
            for b in range(nb):
                n = oh[b + 1] - oh[b]
                _lib.check(lib.dib_mi_sandwich_bounds_batched(_lib.ptr(ml[oh[b]:oh[b + 1]]), 1, n, E, None,
                                                              (int(seed) << 16) + b, 1, _lib.ptr(scratch),
                                                              _lib.ptr(per_set[b]), stream))
                per_set[b] *= n / bs
    return per_set.mean(0).cpu().numpy()


SIMILARITY_TYPES = {"l2sq": 0, "l2": 1, "l1": 2, "linf": 3, "cosine": 4}


def _similarity_kind(similarity_type):
    if similarity_type not in SIMILARITY_TYPES:
        raise ValueError(f"Similarity type not implemented: {similarity_type}")      # utils.py:172
    return SIMILARITY_TYPES[similarity_type]


def get_scaled_similarity(embeddings1, embeddings2, similarity_type, temperature):
    """utils.py:127-175 on the GPU (dib_scaled_similarity): [N, d], [M, d] -> [N, M] similarities / temperature."""
    kind = _similarity_kind(similarity_type)
    if not torch.cuda.is_available():
        raise _lib.DibError("dib_b200 needs a CUDA device; there is no CPU path")
    lib = _lib.load()
    device = (embeddings1.device if isinstance(embeddings1, torch.Tensor) and embeddings1.is_cuda
              else torch.device("cuda", torch.cuda.current_device()))
    e1, e2 = _dev(embeddings1, device), _dev(embeddings2, device)
    if e1.shape[1] != e2.shape[1]:
        raise ValueError("embedding dimensions differ")
    out = torch.empty(e1.shape[0], e2.shape[0], dtype=torch.float32, device=device)
    with torch.cuda.device(device):
        _lib.check(lib.dib_scaled_similarity(kind, _lib.ptr(e1), e1.shape[0], _lib.ptr(e2), e2.shape[0], e1.shape[1],
                                             float(temperature), _lib.ptr(out),
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return out if isinstance(embeddings1, torch.Tensor) else out.cpu().numpy()


def infonce_loss_and_grads(embeddings1, embeddings2, similarity_type, temperature, want_grads=True):
    """The InfoNCE head of the custom loop (train.py:203-213) with its reverse mode (dib_infonce_head).
    Returns (loss [1], d loss/d embeddings1, d loss/d embeddings2) as device tensors (grads None if not wanted)."""
    kind = _similarity_kind(similarity_type)
    lib = _lib.load()
    device = (embeddings1.device if isinstance(embeddings1, torch.Tensor) and embeddings1.is_cuda
              else torch.device("cuda", torch.cuda.current_device()))
    e1, e2 = _dev(embeddings1, device), _dev(embeddings2, device)
    if e1.shape != e2.shape:
        raise ValueError("the InfoNCE loss needs two [n, d] batches of equal shape (train.py:222-223)")
    n, d = e1.shape
    scratch = torch.empty(n * n + 4 * n, dtype=torch.float32, device=device)
    loss = torch.empty(1, dtype=torch.float32, device=device)
    d1 = torch.empty_like(e1) if want_grads else None
    d2 = torch.empty_like(e2) if want_grads else None
    with torch.cuda.device(device):
        _lib.check(lib.dib_infonce_head(kind, _lib.ptr(e1), _lib.ptr(e2), n, d, float(temperature), _lib.ptr(scratch),
                                        _lib.ptr(loss), _lib.ptr(d1), _lib.ptr(d2),
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return loss, d1, d2
