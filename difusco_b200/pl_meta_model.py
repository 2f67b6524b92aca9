"""COMetaModel: the reference's meta model (difusco/pl_meta_model.py) reduced to the inference path.

Kept (same names, arguments, return conventions):
  __init__(param_args, node_feature_only)     :17-47   builds the diffusion tables + GNNEncoder
  categorical_posterior(target_t, t, x0_pred_prob, xt)   :102-146
  gaussian_posterior(target_t, t, pred, xt)              :148-175
  duplicate_edge_index(edge_index, num_nodes, device)    :177-184
plus `posterior_consts`, the float64 host arithmetic of the two posteriors factored out so that the
fused CUDA step (dfb_denoise_step / dfb_denoise) receives four fp32 numbers per step instead of
doing 2x2 inverses and H2D copies every step as the reference does.
Training, optimizers and dataloaders are outside this package's scope.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import _cabi
from .models.gnn_encoder import GNNEncoder
from .utils.diffusion_schedulers import CategoricalDiffusion, GaussianDiffusion

try:   # in a Lightning environment stay a LightningModule so Trainer.test(model) keeps working
  import pytorch_lightning as pl
  _Base = pl.LightningModule
except Exception:   # pragma: no cover - Lightning is not in this image
  class _Base(torch.nn.Module):
    """Stand-in for LightningModule when Lightning is absent: `log` keeps running sums so that `logged_metrics()` gives
    the epoch means Lightning's `on_epoch=True` reduction would report, and `sync_dist=True` (pl_tsp_model.py:253-255,
    pl_mis_model.py:187-192) also averages over the ranks of an initialised process group."""

    def log(self, name, value, prog_bar=False, on_step=None, on_epoch=None, sync_dist=False, **_):
      acc = self.__dict__.setdefault("_dfb_logged", {})
      s = acc.setdefault(name, [0.0, 0, False])
      s[0] += float(value) if not hasattr(value, "__len__") else float(torch.as_tensor(value, dtype=torch.float64).mean())
      s[1] += 1
      s[2] = s[2] or bool(sync_dist)

    def logged_metrics(self, reset=False):
      """{name: mean over the logged steps (and over ranks for sync_dist metrics)}; every rank must call it when a
      process group is initialised and any metric was logged with sync_dist=True (it is a collective then)."""
      import torch.distributed as dist
      acc = self.__dict__.get("_dfb_logged", {})
      out = {}
      use_dist = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
      for name in sorted(acc):
        total, count, sync = acc[name]
        if sync and use_dist:
          dev = torch.device("cuda", torch.cuda.current_device()) if dist.get_backend() == "nccl" else torch.device("cpu")
          t = torch.tensor([total, float(count)], dtype=torch.float64, device=dev)
          dist.all_reduce(t, op=dist.ReduceOp.SUM)
          total, count = float(t[0]), float(t[1])
        out[name] = total / max(count, 1)
      if reset:
        acc.clear()
      return out

    @classmethod
    def load_from_checkpoint(cls, checkpoint_path, map_location=None, strict=True, **kwargs):
      """LightningModule.load_from_checkpoint for the call train.py:127 makes
      (`model_class.load_from_checkpoint(ckpt_path, param_args=args)`): a Lightning .ckpt is a torch pickle whose
      'state_dict' holds this module's keys ('model.' + GNNEncoder.state_dict())."""
      ckpt = torch.load(checkpoint_path, map_location=map_location or "cpu", weights_only=False)
      module = cls(**kwargs)
      module.load_state_dict(ckpt["state_dict"] if "state_dict" in ckpt else ckpt, strict=strict)
      return module


def _arg(args, name, default):
  return getattr(args, name, default)


class COMetaModel(_Base):
  def __init__(self, param_args, node_feature_only=False):
    super().__init__()
    self.args = param_args
    self.diffusion_type = self.args.diffusion_type
    self.diffusion_schedule = self.args.diffusion_schedule
    self.diffusion_steps = self.args.diffusion_steps
    self.sparse = self.args.sparse_factor > 0 or node_feature_only
    if self.diffusion_type == "gaussian":
      out_channels = 1
      self.diffusion = GaussianDiffusion(T=self.diffusion_steps, schedule=self.diffusion_schedule)
    elif self.diffusion_type == "categorical":
      out_channels = 2
      self.diffusion = CategoricalDiffusion(T=self.diffusion_steps, schedule=self.diffusion_schedule)
    else:
      raise ValueError(f"Unknown diffusion type {self.diffusion_type}")
    self.model = GNNEncoder(
        n_layers=self.args.n_layers,
        hidden_dim=self.args.hidden_dim,
        out_channels=out_channels,
        aggregation=self.args.aggregation,
        sparse=self.sparse,
        use_activation_checkpoint=_arg(self.args, "use_activation_checkpoint", False),
        node_feature_only=node_feature_only,
        edge_precision=_arg(self.args, "edge_precision", "bf16x3"),
    )
    self._step_counter = 0

  # ---------------------------------------------------------------------------------------
  # host-side constants of one reverse step
  # ---------------------------------------------------------------------------------------
  def posterior_consts(self, t, target_t):
    """(consts[4] fp32, last flag) for source step t -> target step target_t (ints).

    categorical (pl_meta_model.py:113-137): with Q = inv(Qbar[target]) @ Qbar[t] (float64, then each
    table cast to fp32 as at :115-120) the reference evaluates, through one-hot matmuls,
        p = Q[1,xt] Qbar_tgt[0,1] / Qbar_src[0,xt] * p0[0] + Q[1,xt] Qbar_tgt[1,1] / Qbar_src[1,xt] * p0[1]
    so c[x][k] = (Q[1,x] * Qbar_tgt[k,1]) / Qbar_src[k,x] in fp32, same operation order.
    gaussian (:160-174): xt' = a (xt - b1 pred) + b2 pred + noise z."""
    d = self.diffusion
    t, target_t = int(t), int(target_t)
    if self.diffusion_type == "categorical":
      Q = (np.linalg.inv(d.Q_bar[target_t]) @ d.Q_bar[t]).astype(np.float32)
      src, tgt = d.Q_bar[t].astype(np.float32), d.Q_bar[target_t].astype(np.float32)
      c = [np.float32(Q[1, x] * tgt[k, 1]) / src[k, x] for x in (0, 1) for k in (0, 1)]
      return np.array(c, dtype=np.float32), int(target_t == 0)
    trick = _arg(self.args, "inference_trick", "ddim")
    if trick is None or t <= 1:
      at = d.alpha[t]
      a = (1 / np.sqrt(at)).item()
      b1 = ((1 - at) / np.sqrt(1 - d.alphabar[t])).item()
      noise = np.sqrt(d.beta[t - 1] * (1 - d.alphabar[t - 1]) / (1 - d.alphabar[t])).item()
      return np.array([a, b1, 0.0, noise], dtype=np.float32), 0
    if trick == "ddim":
      a = np.sqrt(d.alphabar[target_t] / d.alphabar[t]).item()
      return np.array([a, np.sqrt(1 - d.alphabar[t]).item(), np.sqrt(1 - d.alphabar[target_t]).item(), 0.0],
                      dtype=np.float32), 0
    raise ValueError("Unknown inference trick {}".format(trick))

  @staticmethod
  def _as_int(t):
    if isinstance(t, torch.Tensor):
      return int(t.reshape(-1)[0].item())
    return int(np.asarray(t).reshape(-1)[0])

  # ---------------------------------------------------------------------------------------
  # reference-signature posteriors (torch ops on whatever device the inputs live on).  The fused
  # denoise steps do NOT go through these; they exist so code that calls them directly keeps working.
  # ---------------------------------------------------------------------------------------
  def categorical_posterior(self, target_t, t, x0_pred_prob, xt):
    t = self._as_int(t)
    target_t = t - 1 if target_t is None else self._as_int(target_t)
    c, last = self.posterior_consts(t, target_t)
    c = torch.from_numpy(c).to(x0_pred_prob.device).reshape(2, 2)
    xi = xt.long().reshape(x0_pred_prob.shape[:-1])
    p = c[xi, 0] * x0_pred_prob[..., 0] + c[xi, 1] * x0_pred_prob[..., 1]
    xt = p.clamp(min=0) if last else torch.bernoulli(p.clamp(0, 1))
    if self.sparse:
      xt = xt.reshape(-1)
    return xt

  def gaussian_posterior(self, target_t, t, pred, xt):
    t = self._as_int(t)
    target_t = t - 1 if target_t is None else self._as_int(target_t)
    (a, b1, b2, noise), _ = self.posterior_consts(t, target_t)
    out = float(a) * (xt - float(b1) * pred) + float(b2) * pred
    if noise != 0.0:
      out = out + float(noise) * torch.randn_like(xt)
    return out

  def duplicate_edge_index(self, edge_index, num_nodes, device):
    """Replicate edge_index parallel_sampling times with +p*num_nodes offsets (:177-184)."""
    P = self.args.parallel_sampling
    ei = edge_index.reshape((2, 1, -1))
    shift = (torch.arange(0, P).view(1, -1, 1).to(device)) * num_nodes
    return (ei + shift).reshape((2, -1))

  # ---------------------------------------------------------------------------------------
  # fused device steps shared by the TSP / MIS task models
  # ---------------------------------------------------------------------------------------
  def _fused_step(self, xt, t, target_t, want_prob=False):
    """One *_denoise_step on the graph already prepared in self.model.  xt: flat float CUDA tensor."""
    ctx = self.model.engine()
    t = self._as_int(t)
    target_t = t - 1 if target_t is None else self._as_int(target_t)
    consts, last = self.posterior_consts(t, target_t)
    dev = xt.device
    n = xt.numel()
    xin = xt.reshape(-1).float().contiguous()
    out = torch.empty(n, device=dev, dtype=torch.float32)
    p = torch.empty(n, device=dev, dtype=torch.float32) if want_prob else None
    if self.diffusion_type == "categorical":
      draws = None if last else torch.rand(n, device=dev, dtype=torch.float32)
      mode = _cabi.CATEGORICAL
    else:
      draws = torch.randn(n, device=dev, dtype=torch.float32) if consts[3] != 0.0 else None
      if consts[3] == 0.0 and t <= 1:
        # the reference draws randn_like(xt) here even though its coefficient is 0 (:164): draw the same number of
        # elements so that torch's generator offset advances exactly as in the reference
        torch.randn(n, device=dev, dtype=torch.float32)
      mode = _cabi.GAUSSIAN
    self._step_counter += 1
    ctx.denoise_step(mode, xin.data_ptr(), float(t), consts, last, draws.data_ptr() if draws is not None else None,
                     0, self._step_counter, out.data_ptr(), p.data_ptr() if p is not None else None, None,
                     torch.cuda.current_stream().cuda_stream)
    return (out, p) if want_prob else out

  def _fused_loop(self, xt, steps, seed=None, record_steps=None, instance_seeds=None):
    """The whole reverse-diffusion loop on device (pl_tsp_model.py:207-217).  In place on xt.

    instance_seeds (a sequence of ints, one per instance of the prepared graph, or per sample of a dense call) keys
    the sampling per instance instead of by the element's index in the call: each instance then draws what it draws
    when denoised alone with seed=instance_seeds[i], whatever else is in the batch.

    record_steps (a list of step indices, or "all") also records those steps from inside the same loop and returns
    (xt, trace): trace["steps"] the recorded step indices, "t" their source timesteps t1, "xt" (n_rec, N) the state
    after each step, "p" (n_rec, N) the categorical p before sampling (categorical only), "out" (n_rec, N,
    out_channels) the network output; all CUDA tensors in xt's element order."""
    from .utils.diffusion_schedulers import InferenceSchedule
    ctx = self.model.engine()
    sched = InferenceSchedule(inference_schedule=self.args.inference_schedule, T=self.diffusion.T,
                              inference_T=steps)
    t1s, consts, lasts = [], [], []
    for i in range(steps):
      t1, t2 = sched(i)
      c, last = self.posterior_consts(int(t1), int(t2))
      t1s.append(int(t1))
      consts.append(c)
      lasts.append(last)
    seeds = None
    if instance_seeds is not None:
      if seed is not None:
        raise ValueError("give seed or instance_seeds, not both")
      seeds = _cabi.instance_seeds_array(instance_seeds, self.model._n_segments)
    elif seed is None:   # honour torch.manual_seed like the reference's torch.bernoulli would
      seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    mode = _cabi.CATEGORICAL if self.diffusion_type == "categorical" else _cabi.GAUSSIAN
    stream = torch.cuda.current_stream().cuda_stream
    rec = []
    if record_steps is not None:
      rec = list(range(steps)) if isinstance(record_steps, str) and record_steps == "all" else \
          [int(s) for s in record_steps]
      if any(s < 0 or s >= steps for s in rec) or any(b <= a for a, b in zip(rec, rec[1:])):
        raise ValueError(f"record_steps must be strictly increasing and inside [0, {steps}): {rec}")
    # pinned and non-blocking: enqueuing a loop never waits for the loops already on the stream
    d_seeds = None if seeds is None else \
        torch.from_numpy(seeds.view(np.int64)).pin_memory().to(xt.device, non_blocking=True)
    if record_steps is None:
      if d_seeds is None:
        ctx.denoise(mode, xt.data_ptr(), t1s, consts, lasts, None, seed, stream)
      else:
        ctx.denoise_instances(mode, xt.data_ptr(), t1s, consts, lasts, d_seeds.data_ptr(), seeds.size, (), None,
                              None, None, stream)
      return xt
    n, dev = xt.numel(), xt.device
    out_channels = 2 if mode == _cabi.CATEGORICAL else 1
    trace = {"steps": torch.tensor(rec, dtype=torch.int64, device=dev),
             "t": torch.tensor([t1s[s] for s in rec], dtype=torch.int64, device=dev),
             "xt": torch.empty((len(rec), n), device=dev, dtype=torch.float32),
             "out": torch.empty((len(rec), n, out_channels), device=dev, dtype=torch.float32)}
    if mode == _cabi.CATEGORICAL:
      trace["p"] = torch.empty((len(rec), n), device=dev, dtype=torch.float32)
    ptrs = (trace["xt"].data_ptr(), trace["p"].data_ptr() if "p" in trace else None, trace["out"].data_ptr())
    if d_seeds is None:
      ctx.denoise_record(mode, xt.data_ptr(), t1s, consts, lasts, rec, *ptrs, None, seed, stream)
    else:
      ctx.denoise_instances(mode, xt.data_ptr(), t1s, consts, lasts, d_seeds.data_ptr(), seeds.size, rec, *ptrs,
                            stream)
    return xt, trace

  # ---------------------------------------------------------------------------------------
  # solving a stream of batches: solve_batch is the one-batch case of solve_batches
  # ---------------------------------------------------------------------------------------
  # Where a batch's 2-opt runs: on a second, higher-priority stream beside the next batch's loops (True), or on the
  # loops' stream, where it follows the next batch's loops already enqueued there (False).  Chosen by measurement
  # (DESIGN §4.2, "Solving a batch"); not an option.
  _two_opt_beside_loop = True

  def solve_batch(self, batch, seeds, split="test"):
    """test_step for every instance of a collated batch at once (see _solve_enqueue of the task model).  seeds: one int
    per instance; instance i's round seeds and initial noise come from a torch.Generator seeded with seeds[i] alone and
    the sampling is keyed per instance, so its result does not depend on the other instances of the batch.  Returns one
    metrics dict per instance with test_step's keys, and logs them as n test_step calls would."""
    return next(self.solve_batches([batch], [seeds], split))

  def solve_batches(self, batches, seeds, split="test"):
    """Generator: for each batch of `batches` (any iterable of collated batches, e.g. a DataLoader), in order, yields
    exactly what solve_batch(batch, seeds[k], split) returns, logs what it logs and sets its last_* artefacts when it
    yields.  seeds: one seed list per batch.

    The host work of one batch is hidden behind the next batch's loops: batch k + 1's inputs are prepared and its
    denoise loops enqueued before batch k is decoded, heat maps reach the host through pinned buffers and events, and
    batch k's 2-opt runs beside batch k + 1's loops.  An exception of batch k (a malformed batch, bad seeds, fewer or
    more seed lists than batches) is raised when batch k is reached, after batches < k were yielded; the model stays
    usable."""
    batches, seed_lists = iter(batches), iter(seeds)
    job = self._next_solve_job(batches, seed_lists)
    while job is not None:
      if isinstance(job, Exception):
        raise job
      following = self._next_solve_job(batches, seed_lists)
      yield self._solve_finish(job, split)
      job = following

  def _next_solve_job(self, batches, seed_lists):
    """_solve_enqueue of the next batch -> its job, None after the last batch, or the exception it raised."""
    end = object()
    try:
      batch, seeds = next(batches, end), next(seed_lists, end)
      if batch is end:
        if seeds is not end:
          raise ValueError("solve_batches: more seed lists than batches")
        return None
      if seeds is end:
        raise ValueError("solve_batches: fewer seed lists than batches")
      return self._solve_enqueue(batch, seeds)
    except Exception as e:   # raised when this batch is reached, after the earlier ones were yielded
      return e

  @staticmethod
  def _pinned_to_device(x, dev):
    """Host tensor -> device copy that does not wait for the work already on the stream."""
    return x.pin_memory().to(dev, non_blocking=True)

  @staticmethod
  def _to_host_async(x):
    """Device tensor -> (pinned host copy, event recorded after the copy); wait on the event before reading it."""
    host = torch.empty(x.shape, dtype=x.dtype, pin_memory=True)
    host.copy_(x, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    return host, ev

  def _two_opt_stream(self, dev):
    """The stream a batch's 2-opt runs on (see _two_opt_beside_loop)."""
    if not self._two_opt_beside_loop:
      return torch.cuda.current_stream(dev)
    s = self.__dict__.get("_dfb_two_opt_stream")
    if s is None or s.device != dev:
      s = torch.cuda.Stream(dev, priority=-1)   # higher priority: its short launches go first at launch boundaries
      self.__dict__["_dfb_two_opt_stream"] = s
    return s

  @staticmethod
  def _solve_seeds(seeds, n):
    """solve_batch's seeds -> n torch.Generators, instance i's seeded with seeds[i] alone."""
    if isinstance(seeds, (str, bytes)) or not hasattr(seeds, "__len__"):
      raise ValueError(f"seeds must be a sequence of integers, got {type(seeds).__name__}")
    if len(seeds) != n:
      raise ValueError(f"{len(seeds)} seeds for {n} instances")
    gens = []
    for s in seeds:
      if isinstance(s, (bool, np.bool_)) or not isinstance(s, (int, np.integer)) or not 0 <= int(s) < 2 ** 63:
        raise ValueError(f"seeds must be integers in [0, 2**63), got {s!r}")
      gens.append(torch.Generator().manual_seed(int(s)))
    return gens

  @staticmethod
  def _round_seed(gen):
    """The Philox seed of one sequential round, drawn from the instance's own generator."""
    return int(torch.randint(0, 2 ** 62, (1,), generator=gen).item())
