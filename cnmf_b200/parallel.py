"""Multi-GPU factorize: restarts shard across ranks, one all-gather of spectra before consensus.

The reference parallelises factorize by launching independent worker processes that take jobs
`(idx - worker_i) % total_workers == 0` and meet again on disk in `combine` (cnmf.py:52-53, 677-689,
748-773; Extras/run_parallel.py).  Here: one process per GPU (torchrun), the same round-robin job
split, the normalised counts replicated on every GPU, and ONE collective -- an all-gather of each
rank's packed spectra slab over NCCL/NVLink -- replacing the trip through the filesystem.  There is no
other exchange on the path (restarts are independent), so scaling is weak in the number of restarts.

Host logic is backend-agnostic (gloo on CPU in the tests, nccl on GPUs).
"""
import os

import numpy as np


def dist_info():
    """(rank, world_size, local_rank) from the torchrun environment (1-process defaults)."""
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")),
            int(os.environ.get("LOCAL_RANK", "0")))


def init_process_group(backend=None):
    import torch
    import torch.distributed as dist
    rank, world, local = dist_info()
    if world == 1:
        return None
    if not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29512")
        kwargs = {}
        if backend == "nccl":
            kwargs["device_id"] = torch.device("cuda:%d" % local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world, **kwargs)
    return dist


def shard_jobs(n_jobs, rank, world):
    """Job indices of this rank: idx % world == rank over the k-major / iter-minor job list
    (same rule as the reference's worker_filter, cnmf.py:52-53), so every K's seeds spread evenly."""
    return [i for i in range(n_jobs) if (i - rank) % world == 0]


_LAYOUTS = {}     # (ks_all, world) -> (rows_per_rank, first_row): the slab layout is a function of the job table only


def _slab_layout(ks_all, world):
    """Rows every rank contributes and the first slab row of every job, for a slab of (world, max_rows) rows.
    Cached: a K-sweep calls factorize_sharded with the same table over and over, and 17 passes of Python over
    900 jobs leave the GPU idle on every call."""
    key = (tuple(ks_all), int(world))
    hit = _LAYOUTS.get(key)
    if hit is None:
        n_jobs = len(ks_all)
        per_rank = [shard_jobs(n_jobs, r, world) for r in range(world)]
        rows_per_rank = [sum(ks_all[j] for j in jobs) for jobs in per_rank]
        max_rows = max(max(rows_per_rank), 1)
        first_row = [0] * n_jobs
        for r, jobs in enumerate(per_rank):
            o = 0
            for j in jobs:
                first_row[j] = r * max_rows + o
                o += ks_all[j]
        if len(_LAYOUTS) > 16:
            _LAYOUTS.clear()
        hit = _LAYOUTS[key] = (rows_per_rank, max_rows, first_row, per_rank)
    return hit


def allgather_spectra(local_spectra, local_jobs, ks_all, n_genes, device=None):
    """All-gather the per-rank spectra slabs and return the list of spectra for ALL jobs, in job order.

    local_spectra : list of (k_j x G) float32 arrays for this rank's jobs (same order as local_jobs)
    ks_all        : k of every job (global list, identical on all ranks)
    Every rank's slab is padded to the largest per-rank row count so one fixed-size all_gather suffices
    (payload: sum(k) * G * 4 bytes in total, e.g. 65 MB at 50k x 2k, K=5..13 x 100)."""
    import torch
    import torch.distributed as dist
    rank, world, _ = dist_info()
    n_jobs = len(ks_all)
    if world == 1 or not dist.is_initialized():
        out = [None] * n_jobs
        for j, s in zip(local_jobs, local_spectra):
            out[j] = np.asarray(s, dtype=np.float32)
        return out
    rows_per_rank = [sum(ks_all[j] for j in shard_jobs(n_jobs, r, world)) for r in range(world)]
    max_rows = max(rows_per_rank)
    use_cuda = dist.get_backend() == "nccl"
    dev = torch.device("cuda:%d" % (device if device is not None else torch.cuda.current_device())) if use_cuda else torch.device("cpu")
    slab = torch.zeros((max_rows, n_genes), dtype=torch.float32, device=dev)
    if local_spectra:
        packed = np.ascontiguousarray(np.vstack(local_spectra), dtype=np.float32)
        slab[: packed.shape[0]].copy_(torch.from_numpy(packed))
    gathered = torch.empty((world * max_rows, n_genes), dtype=torch.float32, device=dev)
    dist.all_gather_into_tensor(gathered, slab)
    host = gathered.cpu().numpy().reshape(world, max_rows, n_genes)
    out = [None] * n_jobs
    for r in range(world):
        o = 0
        for j in shard_jobs(n_jobs, r, world):
            out[j] = host[r, o:o + ks_all[j]].copy()
            o += ks_all[j]
    return out


class SpectraComm:
    """The library's own NCCL communicator (C ABI: cnmf_comm_unique_id / cnmf_comm_create), bootstrapped by shipping
    the 128-byte id through torch.distributed's process group -- the only thing torch.distributed is used for on
    the NCCL path.  A host that already owns an ncclComm_t passes it to cnmf_allgather_spectra directly."""

    def __init__(self, engine):
        import ctypes
        import torch.distributed as dist
        from ._lib import check
        self.engine = engine
        self.lib = engine.lib
        rank, world, _ = dist_info()
        buf = ctypes.create_string_buffer(128)
        if rank == 0:
            check(self.lib.cnmf_comm_unique_id(buf))
        box = [bytes(buf.raw)]
        dist.broadcast_object_list(box, src=0)
        self._comm = ctypes.c_void_p()
        check(self.lib.cnmf_comm_create(engine._h, ctypes.create_string_buffer(box[0], 128), rank, world,
                                        ctypes.byref(self._comm)))

    def allgather(self, local_t, merged_t):
        """merged_t (world x rows x ld) <- every rank's local_t (rows x ld); device tensors, asynchronous."""
        import ctypes
        from ._lib import check
        rows, ld = int(local_t.shape[0]), int(local_t.shape[1])
        check(self.lib.cnmf_allgather_spectra(self._comm, ctypes.c_void_p(local_t.data_ptr()), rows, ld,
                                              ctypes.c_void_p(merged_t.data_ptr()), None))

    def close(self):
        if self._comm:
            self.lib.cnmf_comm_destroy(self._comm)
            import ctypes
            self._comm = ctypes.c_void_p()


_PINNED = {}      # pinned staging buffer of ShardedSpectra.host(), keyed by slab shape


class ShardedSpectra:
    """Result of factorize_sharded: every restart's spectra in ONE device slab (world x max_rows x ld), identical on
    all ranks after the all-gather, plus the map job -> slab row."""

    def __init__(self, gathered, ks_all, n_genes, world):
        self.t = gathered                       # torch tensor (world, max_rows, ld) on the device
        self.ks_all = list(ks_all)
        self.n_genes = int(n_genes)
        self.world = int(world)
        self.max_rows = int(gathered.shape[1])
        self.ld = int(gathered.shape[2])
        _, max_rows, self.first_row, _ = _slab_layout(self.ks_all, self.world)
        assert max_rows == self.max_rows, "slab does not have the layout of this job table"

    def rows_of_jobs(self, jobs):
        """Slab rows (flattened world*max_rows index) of the given jobs, job by job, component by component."""
        out = []
        for j in jobs:
            out.extend(range(self.first_row[j], self.first_row[j] + self.ks_all[j]))
        return np.asarray(out, dtype=np.int32)

    def matrix(self, engine, jobs):
        """The stacked spectra of `jobs` (what `combine` would have merged, cnmf.py:748-773) as a device matrix."""
        from .consensus import SpectraMatrix
        return SpectraMatrix.from_device_rows(engine, self.t.data_ptr(), self.ld, self.rows_of_jobs(jobs), self.n_genes)

    def host(self):
        """All spectra on the host, list indexed by job: ONE contiguous copy of the slab into pinned memory (cached per
        size), then per-job views -- much faster than a pitched copy into pageable memory."""
        import torch
        n = self.world * self.max_rows
        key = (n, self.ld)
        buf = _PINNED.get(key)
        if buf is None:
            _PINNED.clear()
            buf = _PINNED[key] = torch.empty((n, self.ld), dtype=torch.float32, pin_memory=True)
        buf.copy_(self.t.reshape(n, self.ld), non_blocking=True)
        torch.cuda.synchronize(self.t.device)
        flat = buf.numpy()
        return [flat[self.first_row[j]:self.first_row[j] + k, :self.n_genes] for j, k in enumerate(self.ks_all)]


def factorize_sharded(ds, ks_all, seeds_all, nmf_kwargs, comm=None, X_host=None):
    """The multi-GPU factorize: this rank's jobs (idx % world == rank, cnmf.py:52-53) in one batched solve whose
    spectra stay in HBM, then ONE NCCL all-gather of the per-rank slabs (cnmf_allgather_spectra).  No host staging:
    random and NNDSVD starts are computed on the device (X_host: take the NNDSVD starts from the host instead).
    Returns (ShardedSpectra, n_iter of the local jobs, local job indices).  Float64 datasets (precision='fp64') are
    refused: the slabs and the all-gather are float32."""
    if getattr(ds, "fp64", False):
        raise NotImplementedError("cnmf_b200: the sharded multi-GPU factorize gathers float32 spectra; precision='fp64' "
                                  "runs on one GPU per process (cNMF.factorize)")
    import torch
    rank, world, _ = dist_info()
    _, max_rows, _, per_rank = _slab_layout(ks_all, world)
    jobs = per_rank[rank]
    _, ld = ds.ld()
    dev = torch.device("cuda:%d" % ds.engine.device)
    gathered = torch.zeros((world, max_rows, ld), dtype=torch.float32, device=dev)
    slab = gathered[rank] if world == 1 else torch.zeros((max_rows, ld), dtype=torch.float32, device=dev)
    n_iter = np.zeros(0, np.int32)
    if jobs and nmf_kwargs.get("init", "random") != "random" and X_host is not None:
        sp, _, n_iter, _ = ds.factorize([ks_all[j] for j in jobs], [seeds_all[j] for j in jobs], nmf_kwargs, X_host=X_host)
        rows = np.vstack(sp)
        slab[:rows.shape[0], :rows.shape[1]].copy_(torch.from_numpy(rows))
    elif jobs:
        n_iter, _ = ds.factorize_seeds_dev([ks_all[j] for j in jobs], [seeds_all[j] for j in jobs], slab.data_ptr(), ld,
                                           nmf_kwargs)
    if world > 1:
        own = comm is None
        if own:
            comm = SpectraComm(ds.engine)
        comm.allgather(slab, gathered)
        torch.cuda.synchronize(dev)
        if own:
            comm.close()
    return ShardedSpectra(gathered, ks_all, ds.shape[1], world), n_iter, jobs


def consensus_ks_of_rank(ks_sorted, rank, world):
    """K -> GPU assignment of the consensus sweep (`cnmf consensus` / k_selection_plot loop over K,
    cnmf.py:1119-1135, 1278-1291): consensus for one K is a chain of small dependent kernels, so the Ks -- not the
    rows -- are what shards; every rank holds all spectra after the all-gather."""
    return [k for i, k in enumerate(ks_sorted) if i % world == rank]


def factorize_distributed(cnmf_obj, write_files=True):
    """Sharded cNMF.factorize + in-memory combine.  Every rank factorizes its jobs on its own GPU; the
    spectra slabs are all-gathered on the device; rank 0 writes the per-restart and merged files (so `combine` /
    `consensus` find exactly what the reference would have written).  Returns {k: merged R x G float64 DataFrame}."""
    import pandas as pd
    import yaml
    from . import io as cio
    from .io import load_df_from_npz, save_df_to_npz
    rank, world, local = dist_info()
    init_process_group()
    run_params = load_df_from_npz(cnmf_obj.paths["nmf_replicate_parameters"])
    norm = cio.read_matrix(cnmf_obj.paths["normalized_counts"])
    kw = yaml.load(open(cnmf_obj.paths["nmf_run_parameters"]), Loader=yaml.FullLoader)
    ks_all = [int(k) for k in run_params["n_components"]]
    seeds_all = [int(s) for s in run_params["nmf_seed"]]
    ds = cnmf_obj._dataset(norm.X)
    sharded, _, _ = factorize_sharded(ds, ks_all, seeds_all, kw)
    cnmf_obj.last_sharded_spectra = sharded          # consensus can take its matrices from the device slab
    full = sharded.host()
    merged = {}
    for k in sorted(set(ks_all)):
        rows = run_params[run_params.n_components == k].sort_values("iter")
        parts = []
        for idx, p in rows.iterrows():
            df = pd.DataFrame(full[idx].astype(np.float64), index=["iter%d_topic%d" % (p["iter"], t + 1) for t in range(k)],
                              columns=norm.var_names)
            parts.append(df)
            if write_files and rank == 0:
                per = df.copy()
                per.index = np.arange(1, k + 1)
                save_df_to_npz(per, cnmf_obj.paths["iter_spectra"] % (k, p["iter"]))
        m = pd.concat(parts, axis=0)
        merged[k] = m
        if write_files and rank == 0:
            save_df_to_npz(m, cnmf_obj.paths["merged_spectra"] % k)
    return merged
