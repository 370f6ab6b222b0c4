"""``Model`` — the public entry point, same call signatures as the reference for the importance-sampling
path (pyprob/model.py:23-225): ``prior[_results]``, ``posterior[_results]``, ``learn_inference_network``,
``save/load_inference_network``.  MCMC engines, RemoteModel, ParallelModel and on-disk datasets are out of
scope (SURVEY.md section 8) and raise NotImplementedError.
"""
import warnings

import torch

from . import ops, state, util
from .dataset import OnlineDataset
from .distributions import set_shard_first_index
from .empirical import Empirical
from .network import InferenceNetwork as _InferenceNetworkBase, InferenceNetworkFeedForward, InferenceNetworkLSTM
from .offline import OfflineDataset
from .util import InferenceEngine, InferenceNetwork, LearningRateScheduler, Optimizer, PriorInflation, TraceMode


def trace_result(trace):
    return trace.result


class Model:
    def __init__(self, name='Unnamed PyProb model', address_dict_file_name=None):
        self.name = name
        self._inference_network = None
        self._scalar_mode = False  # True once a batched execution hit python-scalar control flow
        if address_dict_file_name is not None:
            raise NotImplementedError('address dictionaries are out of scope for pyprob_b200')

    def __repr__(self):
        return 'Model(name:{})'.format(self.name)

    def forward(self):
        raise RuntimeError('Model instances must provide a forward method.')

    # ---- execution ------------------------------------------------------------------------------------------
    def _run_batched(self, n, trace_mode=TraceMode.PRIOR, prior_inflation=PriorInflation.DISABLED,
                     inference_engine=InferenceEngine.IMPORTANCE_SAMPLING, inference_network=None, observe=None,
                     likelihood_importance=1.0, init=True, *args, **kwargs):
        """Run ``forward`` once for n particles in lock-step and return the BatchedTrace."""
        if init:
            state._init_traces(self.forward, trace_mode=trace_mode, prior_inflation=prior_inflation,
                               inference_engine=inference_engine, inference_network=inference_network, observe=observe,
                               likelihood_importance=likelihood_importance)
        state._begin_trace(n)
        try:
            result = self.forward(*args, **kwargs)
        except Exception:
            state._current_trace = None
            raise
        return state._end_trace(result)

    def _traces(self, num_traces=10, trace_mode=TraceMode.PRIOR, prior_inflation=PriorInflation.DISABLED,
                inference_engine=InferenceEngine.IMPORTANCE_SAMPLING, inference_network=None, map_func=None,
                observe=None, likelihood_importance=1.0, batch_size=None, first_index=0, sharded=False, *args,
                **kwargs):
        """Importance-sampling driver (reference: model.py:47-88) -> Empirical of map_func(trace) values.

        sharded=True (with torch.distributed initialised): `num_traces` is the GLOBAL particle count, this rank
        draws its contiguous index range of the Philox stream and the returned Empirical is normalised globally."""
        if map_func is None:
            map_func = trace_result
        if sharded:
            from . import parallel
            world, rank = parallel.world_info()
            first_index, num_traces = parallel.shard_range(num_traces, rank, world)
        chunk = batch_size or min(num_traces, 1 << 20)
        if self._scalar_mode:
            chunk = 1
        values, weights = [], []
        done = 0
        state._init_traces(self.forward, trace_mode=trace_mode, prior_inflation=prior_inflation,
                           inference_engine=inference_engine, inference_network=inference_network, observe=observe,
                           likelihood_importance=likelihood_importance)
        while done < num_traces:
            n = min(chunk, num_traces - done)
            set_shard_first_index(first_index + done)
            try:
                trace = self._run_batched(n, init=False, *args, **kwargs)
            except (ValueError, RuntimeError) as e:
                if n > 1 and (('convert' in str(e) and 'calar' in str(e)) or 'ambiguous' in str(e)):
                    warnings.warn('Model uses python-scalar control flow on sampled values; running one particle per '
                                  'execution (slow). Use pyprob_b200.while_loop for lock-step loops.')
                    self._scalar_mode, chunk = True, 1
                    continue
                raise
            v = map_func(trace)
            v = v if torch.is_tensor(v) else torch.as_tensor(v, dtype=torch.float32, device='cuda')
            values.append(v.reshape(n, -1) if v.numel() >= n else v.reshape(1, -1).expand(n, -1))
            weights.append(trace.log_w)
            done += n
        set_shard_first_index(0)
        vals = torch.cat(values, dim=0).squeeze(-1)
        acc = torch.cat(weights, dim=0)
        if trace_mode == TraceMode.PRIOR:
            return Empirical(vals, None)
        log_w, bad = ops.weights_cast(acc)
        nbad = int(bad.sum())
        if nbad:  # reference: model.py:65-68 discards traces with NaN / +-inf weights
            warnings.warn('Encountered {} trace(s) with nan, inf, or -inf log_weight. Discarding.'.format(nbad))
            keep = bad == 0
            vals, log_w = vals[keep], log_w[keep]
        return Empirical(vals, log_w, sharded=sharded)

    # ---- public API -------------------------------------------------------------------------------------------
    def prior(self, num_traces=10, prior_inflation=PriorInflation.DISABLED, map_func=None, *args, **kwargs):
        prior = self._traces(num_traces, trace_mode=TraceMode.PRIOR, prior_inflation=prior_inflation,
                             map_func=map_func, *args, **kwargs)
        prior.rename('Prior, traces: {:,}'.format(prior.length))
        return prior

    def prior_results(self, num_traces=10, prior_inflation=PriorInflation.DISABLED, map_func=trace_result, *args,
                      **kwargs):
        return self.prior(num_traces, prior_inflation=prior_inflation, map_func=map_func, *args, **kwargs)

    def posterior(self, num_traces=10, inference_engine=InferenceEngine.IMPORTANCE_SAMPLING, initial_trace=None,
                  map_func=None, observe=None, file_name=None, thinning_steps=None, likelihood_importance=1.,
                  *args, **kwargs):
        if file_name is not None:
            raise NotImplementedError('disk-backed Empiricals are out of scope for pyprob_b200')
        if inference_engine == InferenceEngine.IMPORTANCE_SAMPLING:
            post = self._traces(num_traces, trace_mode=TraceMode.POSTERIOR, inference_engine=inference_engine,
                                map_func=map_func, observe=observe, likelihood_importance=likelihood_importance,
                                *args, **kwargs)
            post.rename('Posterior, IS, traces: {:,}, ESS: {:,.2f}'.format(post.length, post.effective_sample_size))
        elif inference_engine == InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK:
            if self._inference_network is None:
                raise RuntimeError('Cannot run inference engine IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK because no '
                                   'inference network for this model is available. Use learn_inference_network or '
                                   'load_inference_network first.')
            with torch.no_grad():
                post = self._traces(num_traces, trace_mode=TraceMode.POSTERIOR, inference_engine=inference_engine,
                                    inference_network=self._inference_network, map_func=map_func, observe=observe,
                                    likelihood_importance=likelihood_importance, *args, **kwargs)
            post.rename('Posterior, IC, traces: {:,}, train. traces: {:,}, ESS: {:,.2f}'.format(
                post.length, self._inference_network._total_train_traces, post.effective_sample_size))
        else:
            raise NotImplementedError('pyprob_b200 implements IMPORTANCE_SAMPLING and '
                                      'IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK; MCMC engines are out of scope')
        post.add_metadata(op='posterior', num_traces=num_traces, inference_engine=str(inference_engine),
                          effective_sample_size=post.effective_sample_size)
        return post

    def posterior_results(self, num_traces=10, inference_engine=InferenceEngine.IMPORTANCE_SAMPLING,
                          initial_trace=None, map_func=trace_result, observe=None, file_name=None, thinning_steps=None,
                          *args, **kwargs):
        return self.posterior(num_traces, inference_engine=inference_engine, initial_trace=initial_trace,
                              map_func=map_func, observe=observe, file_name=file_name, thinning_steps=thinning_steps,
                              *args, **kwargs)

    def reset_inference_network(self):
        self._inference_network = None

    def learn_inference_network(self, num_traces, num_traces_end=1e9, inference_network=InferenceNetwork.FEEDFORWARD,
                                prior_inflation=PriorInflation.DISABLED, dataset_dir=None, dataset_valid_dir=None,
                                observe_embeddings={}, batch_size=64, valid_size=None, valid_every=None,
                                optimizer_type=Optimizer.ADAM, learning_rate_init=0.001, learning_rate_end=1e-6,
                                learning_rate_scheduler_type=LearningRateScheduler.NONE, momentum=0.9, weight_decay=0.,
                                save_file_name_prefix=None, save_every_sec=600, pre_generate_layers=False,
                                distributed_backend=None, distributed_params_sync_every_iter=10000,
                                distributed_num_buckets=None, dataloader_offline_num_workers=0, stop_with_bad_loss=True,
                                log_file_name=None, lstm_dim=512, lstm_depth=1, proposal_mixture_components=10):
        names = list(observe_embeddings)   # dict (or set) of observable names
        if dataset_dir is None:
            dataset = OnlineDataset(model=self, prior_inflation=prior_inflation)
        else:
            dataset = OfflineDataset(dataset_dir, verbose=True)
            dataset.select_observables(names if names else dataset.observe_names)
        dataset_valid = None
        if dataset_valid_dir is not None:
            dataset_valid = OfflineDataset(dataset_valid_dir, verbose=True)
            dataset_valid.select_observables(names if names else dataset_valid.observe_names)
        if self._inference_network is None:
            print('Creating new inference network...')
            if inference_network == InferenceNetwork.FEEDFORWARD:   # reference model.py:199-200
                self._inference_network = InferenceNetworkFeedForward(
                    model=self, observe_embeddings=observe_embeddings,
                    proposal_mixture_components=proposal_mixture_components)
            elif inference_network == InferenceNetwork.LSTM:
                self._inference_network = InferenceNetworkLSTM(model=self, observe_embeddings=observe_embeddings,
                                                               lstm_dim=lstm_dim, lstm_depth=lstm_depth,
                                                               proposal_mixture_components=proposal_mixture_components)
            else:
                raise ValueError('Unknown inference_network: {}'.format(inference_network))
            if pre_generate_layers:
                if dataset_valid is not None:
                    self._inference_network._pre_generate_layers(dataset_valid, batch_size=batch_size,
                                                                 save_file_name_prefix=save_file_name_prefix)
                self._inference_network._pre_generate_layers(dataset, batch_size=batch_size,
                                                             save_file_name_prefix=save_file_name_prefix)
        else:
            print('Continuing to train existing inference network...')
        self._inference_network.optimize(
            num_traces=num_traces, dataset=dataset, dataset_valid=dataset_valid, num_traces_end=num_traces_end,
            batch_size=batch_size, valid_every=valid_every, optimizer_type=optimizer_type,
            learning_rate_init=learning_rate_init, learning_rate_end=learning_rate_end,
            learning_rate_scheduler_type=learning_rate_scheduler_type, momentum=momentum, weight_decay=weight_decay,
            save_file_name_prefix=save_file_name_prefix, save_every_sec=save_every_sec,
            distributed_backend=distributed_backend,
            distributed_params_sync_every_iter=distributed_params_sync_every_iter,
            distributed_num_buckets=distributed_num_buckets,
            dataloader_offline_num_workers=dataloader_offline_num_workers, stop_with_bad_loss=stop_with_bad_loss,
            log_file_name=log_file_name)

    def save_dataset(self, dataset_dir, num_traces, num_traces_per_file, prior_inflation=PriorInflation.DISABLED,
                     observe_names=None, batch_size=None):
        """Write prior traces as columnar trace files (reference Model.save_dataset, model.py:226-231).  All named
        variables of the model are stored as observables unless ``observe_names`` restricts them."""
        dataset = OnlineDataset(model=self, prior_inflation=prior_inflation)
        if observe_names is None:
            observe_names = [name for name in dataset.example_trace().named_variables]
        return dataset.save_dataset(dataset_dir, num_traces, num_traces_per_file, observe_names, batch_size=batch_size)

    def save_inference_network(self, file_name):
        if self._inference_network is None:
            raise RuntimeError('The model has no trained inference network.')
        self._inference_network._save(file_name)

    def load_inference_network(self, file_name):
        self._inference_network = _InferenceNetworkBase._load(file_name)   # whichever network class was saved
        self._inference_network._model = self
