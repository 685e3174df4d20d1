"""Aggregation server (reference ``Aggregation``, src/aggregation.py:8-190).

``aggregate_updates`` = Robust-LR sign vote + {FedAvg | coordinate median | sign majority} + optional noise + server
step, executed by ONE fused kernel over the flat parameter vector (``ops.fused_aggregate`` in-process, or
``parallel.FusedAggregator`` across GPUs) instead of the reference's ~30 elementwise fp64 passes (SURVEY.md 2.4b).
With ``--select krum | multikrum`` a selection stage runs first: the participants' pairwise update distances
(``ops.pairwise_sqdist``), Krum scores on the host (``ops.krum_select``), and only the admitted participants enter the step.
``--aggr fltrust`` and ``--aggr rfa`` are the same weighted-mean launch with weights from a per-participant pass: FLTrust's trust
scores (``ops.trust_stats``) or RFA's smoothed Weiszfeld weights (``ops.rfa`` over ``ops.rfa_sqdist`` passes).  ``--aggr flame`` is
that launch too: the Gram matrix of the updates (``ops.pairwise_gram``) gives FLAME's cosine clustering, median-norm clip scales and
noise (``ops.flame_admit``), and the admitted participants' clipped updates are averaged with equal weights.
The reference's dead / disabled pieces are available behind flags: ``clip_updates`` (``--server_clip``) and the
diagnostics ``plot_norms`` / ``comp_diag_fisher`` / ``plot_sign_agreement`` (``--diagnostics``), the latter with the
reference's latent bugs fixed (model built on the right device; Fisher uses log-probabilities -- SURVEY.md quirk 7).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from . import ops
from .models.graph import GraphNet


def server_opt_spec(args):
    """``ops.ServerOptState`` keyword arguments of the ``--server_opt*`` flags."""
    return dict(kind=getattr(args, "server_opt", "sgd"), beta1=getattr(args, "server_beta1", 0.9),
                beta2=getattr(args, "server_beta2", 0.99), tau=getattr(args, "server_tau", 1e-3))


class Aggregation:
    def __init__(self, agent_data_sizes, n_params, poisoned_val, args, writer=None, layout=None, fused=None):
        self.agent_data_sizes = agent_data_sizes
        self.args = args
        self.writer = writer
        self.server_lr = args.server_lr
        self.n_params = n_params
        self.poisoned_val = poisoned_val
        self.layout = layout
        self.fused = fused            # parallel.FusedAggregator or None (pure in-process use)
        self.cum_net_mov = 0.0
        self.last_flipped = 0
        self.last_admitted = None     # agent ids admitted by --select (and trusted by --aggr fltrust) in the last round
        self.last_select = None       # the Select/* scalars of the last round
        self.last_trust = None        # the Trust/* scalars of the last round (--aggr fltrust)
        self.last_rfa = None          # the RFA/* scalars of the last round (--aggr rfa)
        self.last_flame = None        # the FLAME/* scalars of the last round (--aggr flame)
        self.opt = None               # full-length server optimizer state of the in-process form (allocated on first use)

    # ---- the server step ------------------------------------------------------------------------------------
    def aggregate_updates(self, w_global, agent_params, cur_round, n_vote=None, root_params=None):
        """In-process form: ``agent_params`` = {agent_id: flat local parameters}.  Updates ``w_global`` in place.  ``root_params``:
        the server's root-trained parameters, needed by ``--aggr fltrust``."""
        ids = list(agent_params.keys())
        ws = [agent_params[i] for i in ids]
        nv = n_vote if n_vote is not None else (self.layout.n_vote if self.layout else None)
        if self._fltrust and root_params is None:
            raise ValueError("--aggr fltrust needs the server's root parameters (root_params)")
        clip = self._clip_scales(ops.update_norms(w_global, ws, nv)) if self._server_clip else None
        all_ids, all_ws = ids, ws
        distances = lambda: ops.pairwise_sqdist(ws, nv if nv is not None else w_global.numel(), w_global if clip is not None else None,
                                                clip)
        rfa_pass = lambda b, members: ops.rfa_sqdist(
            [ws[j] for j in members], b, nv, w_global if clip is not None else None,
            clip[torch.as_tensor(members, device=clip.device)] if clip is not None else None)
        gram = lambda members: ops.pairwise_gram([ws[j] for j in members], w_global, nv)
        keep, weights, scales, total, noise_std = self._admission(ids, clip, distances,
                                                                  lambda: ops.trust_stats(ws, root_params, w_global, nv), rfa_pass, gram,
                                                                  cur_round)
        if keep is not None and len(keep) < len(ids):
            ids, ws, weights = [ids[j] for j in keep], [ws[j] for j in keep], [weights[j] for j in keep]
            scales = scales[torch.as_tensor(keep, device=scales.device)] if scales is not None else None
        prev = w_global.clone() if self.args.diagnostics else None
        flipped = torch.zeros(1, dtype=torch.int64, device=w_global.device)
        if self.opt is None:
            self.opt = ops.ServerOptState(n=w_global.numel(), device=w_global.device, **server_opt_spec(self.args))
        ops.fused_aggregate(w_global, ws, weights, self._mode, self.args.robustLR_threshold, self.server_lr, noise_std, self.args.seed,
                            cur_round,
                            n_vote if n_vote is not None else (self.layout.n_vote if self.layout else None),
                            scales, out=w_global, flipped=flipped, opt=self.opt, total_weight=total)
        self.last_flipped = flipped
        if self.args.diagnostics:
            self.plot_norms(dict(zip(all_ids, ops.update_norms(prev, all_ws, nv).tolist())), cur_round)
            self.plot_sign_agreement(prev, w_global, ws, ids, cur_round)     # the vote that happened: admitted participants only
        return

    def aggregate_slots(self, participants, cur_round):
        """Engine form: participant j's parameters live in ``fused.slot_owner(j)``; updates every rank's global.  Under
        ``--aggr fltrust`` the server's root job is position ``len(participants)``."""
        K = len(participants)
        diag = bool(self.args.diagnostics)
        norms = self.fused.update_norms(K) if self._server_clip or diag else None
        clip = self._clip_scales(norms) if self._server_clip else None
        copies, gathered = None, None
        if (self._select or self._fltrust or self._flame or (self._rfa and self.args.rfa_iters > 0)) and self.fused.gathers(K):
            # on the gather transport every pass reads the same all-gathered copies (one all_gather per round; the root job included)
            gathered = self.fused.gather_participants(K + 1 if self._fltrust else K)
            copies = gathered[:K]
        keep, weights, scales, total, noise_std = self._admission(
            participants, clip, lambda: self.fused.pairwise_sqdist(K, clip, copies), lambda: self.fused.trust_stats(K, K, gathered),
            lambda b, members: self.fused.rfa_sqdist(K, b, clip, members, copies),
            lambda members: self.fused.pairwise_gram(K, members, copies), cur_round)
        if diag:   # the sign-agreement analysis needs the pre-step global parameters and every admitted participant's parameters
            prev = self.fused.w_global.clone()
            ws = [w.clone() for w in self.fused.gather_participants(K)]
            voters = participants
            if keep is not None:
                ws, voters = [ws[j] for j in keep], [participants[j] for j in keep]
        self.fused.aggregate(weights, self._mode, self.args.robustLR_threshold, self.server_lr, noise_std, self.args.seed, cur_round,
                             scales, members=keep, participants=copies, total_weight=total)
        self.last_flipped = self.fused.flipped
        if diag:
            self.plot_norms(dict(zip(participants, norms.tolist())), cur_round)
            self.plot_sign_agreement(prev, self.fused.w_global, ws, voters, cur_round)

    @property
    def _server_clip(self):
        return bool(getattr(self.args, "server_clip", False)) and self.args.clip > 0

    @property
    def _select(self):
        return getattr(self.args, "select", "none") != "none"

    def _admission(self, ids, clip, distances, trust_stats, rfa_pass, gram, cur_round):
        """Admission of the participants ``ids`` shared by both forms of the step: Krum / Multi-Krum on ``distances()`` (``--select``),
        then FLTrust on ``trust_stats()`` (``--aggr fltrust``), RFA's weights from ``rfa_pass(b, members)`` (``--aggr rfa``) or FLAME on
        the Gram matrix ``gram(members)`` (``--aggr flame``).  ``clip``: the server-clipping scales or None.  Returns
        ``(members, weights, scales, total_weight, noise_std)`` for the step: members None admits everyone; weights are per position in
        ``ids``."""
        keep = self._admit(distances(), ids, cur_round) if self._select else None
        noise_std = self.args.noise * self.args.clip
        if self._fltrust:
            return (*self._trust(trust_stats(), ids, keep, cur_round), noise_std)
        if self._flame:
            return self._flame_step(ids, keep, gram, cur_round)
        weights = [float(self.agent_data_sizes[i]) for i in ids]
        if self._rfa:
            return (*self._rfa_weights(ids, keep, weights, clip, rfa_pass, cur_round), noise_std)
        return keep, weights, clip, None, noise_std

    def _admit(self, D, ids, cur_round):
        """Krum / Multi-Krum admission from the pairwise distances ``D`` of the participants ``ids``: the admitted positions
        (ascending).  Records ``last_admitted`` and logs how many corrupt participants (ids < num_corrupt) came and got through."""
        keep = ops.krum_select(D, ids, self.args.select_f, self.args.select_m)
        self.last_admitted = [ids[j] for j in keep]
        nc = self.args.num_corrupt
        self.last_select = {"Select/Corrupt_Participants": sum(1 for i in ids if i < nc),
                            "Select/Corrupt_Admitted": sum(1 for i in self.last_admitted if i < nc)}
        if self.writer is not None:
            for k, v in self.last_select.items():
                self.writer.add_scalar(k, v, cur_round)
        return keep

    @property
    def _fltrust(self):
        return self.args.aggr == "fltrust"

    @property
    def _rfa(self):
        return self.args.aggr == "rfa"

    @property
    def _flame(self):
        return self.args.aggr == "flame"

    @property
    def _mode(self):
        """The aggregate kernel's rule: FLTrust is its weighted mean with trust weights and per-participant scales, RFA with its
        Weiszfeld weights, FLAME with equal weights and its clip scales."""
        return "avg" if self._fltrust or self._rfa or self._flame else self.args.aggr

    def _flame_step(self, ids, keep, gram, cur_round):
        """FLAME over the positions ``keep`` that selection admitted (all when None): ``ops.flame_admit`` on ``gram(candidates)``.
        Returns ``(members, weights, scales, total_weight, noise_std)`` for the step: the admitted positions with weight 1 each, total
        weight their count, the clip scales and noise std ``flame_lambda * S`` -- or, when nobody is admitted, every candidate with weight 0
        and total weight 1, so the aggregate is 0 plus noise.  Records ``last_admitted`` and logs the admitted count, the corrupt ones
        among them (ids < num_corrupt), the clip bound S and the noise std."""
        K = len(ids)
        cand = list(range(K)) if keep is None else [int(j) for j in keep]
        adm, sc, S, noise_std = ops.flame_admit(gram(cand), [ids[j] for j in cand], self.args.flame_lambda)
        members = [cand[j] for j in adm]
        scales = torch.ones(K, dtype=torch.float32)
        scales[torch.as_tensor(cand, dtype=torch.int64)] = sc
        weights, total = [1.0] * K, float(len(members))
        self.last_admitted = [ids[j] for j in members]
        if not members:
            members, weights, total = cand, [0.0] * K, 1.0
        nc = self.args.num_corrupt
        self.last_flame = {"FLAME/Admitted": len(self.last_admitted),
                           "FLAME/Corrupt_Admitted": sum(1 for i in self.last_admitted if i < nc),
                           "FLAME/Clip_Bound": S, "FLAME/Noise_Std": noise_std}
        if self.writer is not None:
            for k, v in self.last_flame.items():
                self.writer.add_scalar(k, v, cur_round)
        return members, weights, scales, total, noise_std

    def _rfa_weights(self, ids, keep, weights, clip, rfa_pass, cur_round):
        """RFA over the positions ``keep`` that selection admitted (all when None): ``--rfa_iters`` smoothed Weiszfeld passes
        (``ops.rfa``) from the data sizes ``weights``, each pass ``rfa_pass(b, members)`` returning the members' squared distances to
        their ``b``-weighted mean.  Nobody is dropped.  Returns ``(members, weights, scales, total_weight)`` for the step: the members'
        weights replaced by the final beta and total weight sum beta (``--rfa_iters 0``: exactly the avg step's weights and total).
        Logs the share of the weight that corrupt participants (ids < num_corrupt) hold."""
        cand = list(range(len(ids))) if keep is None else [int(j) for j in keep]
        T = int(self.args.rfa_iters)
        beta, _ = ops.rfa([weights[j] for j in cand], lambda b: rfa_pass(b, cand), T, self.args.rfa_nu)
        weights = list(weights)
        for j, bj in zip(cand, beta):
            weights[j] = bj
        total = sum(beta)
        nc = self.args.num_corrupt
        self.last_rfa = {"RFA/Corrupt_Weight": sum(bj for j, bj in zip(cand, beta) if ids[j] < nc) / total, "RFA/Passes": T}
        if self.writer is not None:
            for k, v in self.last_rfa.items():
                self.writer.add_scalar(k, v, cur_round)
        return keep, weights, clip, total

    def _trust(self, stats, ids, keep, cur_round):
        """FLTrust admission from the statistics ``stats`` (``ops.trust_statement``'s layout) of the participants ``ids``, among the
        positions ``keep`` that selection admitted (all when None).  Returns ``(members, weights, scales, total_weight)`` for the step:
        the trusted positions (TS > 0) with weights TS, scales s and total weight sum TS -- or, when nobody is trusted, every candidate
        with weight 0 and total weight 1, so the aggregate is 0 (plus noise) and the round still runs its one aggregate launch.
        Records ``last_admitted`` and logs the mean trust of honest (ids >= num_corrupt) and corrupt participants."""
        K = len(ids)
        s = stats.detach().double().cpu()
        ts, scales, _ = ops.fltrust_weights(s[:K], s[K:2 * K], s[2 * K])
        cand = list(range(K)) if keep is None else [int(j) for j in keep]
        members = [j for j in cand if ts[j] > 0]
        weights = [float(ts[j]) for j in range(K)]
        total = sum(weights[j] for j in members)
        if not members:
            members, total = cand, 1.0
            weights = [0.0] * K
        self.last_admitted = [ids[j] for j in cand if ts[j] > 0]
        nc = self.args.num_corrupt
        honest = [float(ts[j]) for j in cand if ids[j] >= nc]
        corrupt = [float(ts[j]) for j in cand if ids[j] < nc]
        self.last_trust = {"Trust/Avg_Honest": sum(honest) / len(honest) if honest else None,
                           "Trust/Avg_Corrupt": sum(corrupt) / len(corrupt) if corrupt else None,
                           "Trust/Admitted": len(self.last_admitted)}
        if self.writer is not None:
            for k, v in self.last_trust.items():
                if v is not None:
                    self.writer.add_scalar(k, v, cur_round)
        return members, weights, scales, total

    def _clip_scales(self, norms):
        """reference ``clip_updates`` (src/aggregation.py:77-81): update /= max(1, ||update||/clip)."""
        return (1.0 / torch.clamp(norms / self.args.clip, min=1.0)).float()

    # ---- reference-named helpers (thin wrappers over the oracle; kept for API parity and tests) -----------------
    def compute_robustLR(self, agent_updates_dict):
        """±server_lr per coordinate from the sign vote (src/aggregation.py:48-54)."""
        s = sum(torch.sign(u) for u in agent_updates_dict.values()).abs()
        return torch.where(s >= self.args.robustLR_threshold, self.server_lr, -self.server_lr).to(s.dtype)

    def agg_avg(self, agent_updates_dict):
        tot = sum(self.agent_data_sizes[i] for i in agent_updates_dict)
        return sum(self.agent_data_sizes[i] * u for i, u in agent_updates_dict.items()) / tot

    def agg_comed(self, agent_updates_dict):
        return torch.median(torch.stack(list(agent_updates_dict.values()), dim=1), dim=1).values

    def agg_sign(self, agent_updates_dict):
        return torch.sign(sum(torch.sign(u) for u in agent_updates_dict.values()))

    def clip_updates(self, agent_updates_dict):
        for u in agent_updates_dict.values():
            u.div_(max(1.0, float(torch.norm(u, p=2)) / self.args.clip))

    # ---- diagnostics ---------------------------------------------------------------------------------------
    def plot_norms(self, norms_by_agent, cur_round, norm=2):
        """Average update norm of honest vs corrupt agents (src/aggregation.py:83-100)."""
        honest = [v for k, v in norms_by_agent.items() if k >= self.args.num_corrupt]
        corrupt = [v for k, v in norms_by_agent.items() if k < self.args.num_corrupt]
        out = {}
        if honest:
            out[f"Norms/Avg_Honest_L{norm}"] = sum(honest) / len(honest)
        if corrupt:
            out[f"Norms/Avg_Corrupt_L{norm}"] = sum(corrupt) / len(corrupt)
        for k, v in out.items():
            if self.writer is not None:
                self.writer.add_scalar(k, v, cur_round)
        self.last_norms = out
        return out

    def comp_diag_fisher(self, model_params, dataset, adv=True, bs=256):
        """Diagonal Fisher information of the log-likelihood of the (adversarial or base-class) label on the poisoned
        validation set (src/aggregation.py:102-129, with quirk 7 fixed)."""
        dev = model_params.device
        w = model_params.clone()
        g = torch.zeros_like(w)
        net = GraphNet(self.layout, w, g)
        net.eval()
        fisher = torch.zeros_like(w)
        n = len(dataset)
        for start in range(0, n, bs):
            idx = torch.arange(start, min(n, start + bs), device=dev)
            x, y = dataset.batch(idx)
            if not adv:
                y = torch.full_like(y, self.args.base_class)
            g.zero_()
            logp = F.log_softmax(net(x), dim=1)
            logp.gather(1, y[:, None]).sum().backward()
            fisher += g ** 2 / n
        return fisher[: self.layout.n_vote].detach()

    def plot_sign_agreement(self, cur_global_params, new_global_params, agent_params, ids, cur_round):
        """Which of the most backdoor-relevant coordinates (top-``top_frac`` Fisher) had their LR kept vs flipped, for
        adversarial vs honest objectives; logs the 7 ``Sign/*`` scalars (src/aggregation.py:132-190)."""
        if self.layout is None or self.poisoned_val is None or len(self.poisoned_val) == 0:
            return {}
        nv = self.layout.n_vote
        update = (new_global_params - cur_global_params)[:nv]
        signs = sum(torch.sign(w[:nv] - cur_global_params[:nv]) for w in agent_params).abs()
        theta = self.args.robustLR_threshold
        lr = torch.where(signs >= theta, 1.0, -1.0) if theta > 0 else torch.ones_like(signs)
        fa = self.comp_diag_fisher(cur_global_params, self.poisoned_val, adv=True)
        fh = self.comp_diag_fisher(cur_global_params, self.poisoned_val, adv=False)
        k = int(self.args.top_frac)
        adv_top = fa.topk(k).indices.cpu().numpy()
        hon_top = fh.topk(k).indices.cpu().numpy()
        min_idxs = (lr < 0).nonzero().flatten().cpu().numpy()
        max_idxs = (lr > 0).nonzero().flatten().cpu().numpy()
        max_adv, max_hon = np.intersect1d(adv_top, max_idxs), np.intersect1d(hon_top, max_idxs)
        min_adv, min_hon = np.intersect1d(adv_top, min_idxs), np.intersect1d(hon_top, min_idxs)
        l2 = lambda ix: float(torch.norm(update[torch.as_tensor(ix, dtype=torch.int64, device=update.device)])) if len(ix) else 0.0
        v = {
            "Sign/Hon_Maxim_L2": l2(np.setdiff1d(max_hon, max_adv)), "Sign/Adv_Maxim_L2": l2(np.setdiff1d(max_adv, max_hon)),
            "Sign/Adv_Minim_L2": l2(np.setdiff1d(min_adv, min_hon)), "Sign/Hon_Minim_L2": l2(np.setdiff1d(min_hon, min_adv)),
        }
        v["Sign/Adv_Net_L2"] = v["Sign/Adv_Maxim_L2"] - v["Sign/Adv_Minim_L2"]
        v["Sign/Hon_Net_L2"] = v["Sign/Hon_Maxim_L2"] - v["Sign/Hon_Minim_L2"]
        self.cum_net_mov += v["Sign/Hon_Net_L2"] - v["Sign/Adv_Net_L2"]
        v["Sign/Model_Net_L2_Cumulative"] = self.cum_net_mov
        for key, val in v.items():
            if self.writer is not None:
                self.writer.add_scalar(key, val, cur_round)
        self.last_sign_stats = v
        return v
