"""Aggregation server (reference ``Aggregation``, src/aggregation.py:8-190).

``aggregate_updates`` = Robust-LR sign vote + {FedAvg | coordinate median | sign majority} + optional noise + server
step, executed by ONE fused kernel over the flat parameter vector (``ops.fused_aggregate`` in-process, or
``parallel.FusedAggregator`` across GPUs) instead of the reference's ~30 elementwise fp64 passes (SURVEY.md 2.4b).
With ``--select krum | multikrum`` a selection stage runs first: the participants' pairwise update distances
(``ops.pairwise_sqdist``), Krum scores on the host (``ops.krum_select``), and only the admitted participants enter the step.
``--select dnc`` is that stage on DnC's spectral scores: the Gram matrices of the updates centred at random coordinate subsamples
(``ops.dnc_grams``), and on the host the top eigenvector's outlier scores and the intersection of the kept sets (``ops.dnc_select``).
``--aggr fltrust`` and ``--aggr rfa`` are the same weighted-mean launch with weights from a per-participant pass: FLTrust's trust
scores (``ops.trust_stats``) or RFA's smoothed Weiszfeld weights (``ops.rfa`` over ``ops.rfa_sqdist`` passes).  ``--aggr flame`` is
that launch too: the Gram matrix of the updates (``ops.pairwise_gram``) gives FLAME's cosine clustering, median-norm clip scales and
noise (``ops.flame_admit``), and the admitted participants' clipped updates are averaged with equal weights.  ``--aggr foolsgold`` keeps
every agent's summed updates across rounds (``ops.history_accumulate``) and weights the mean by FoolsGold's ``ops.foolsgold_weights`` on
the Gram matrix of those histories (``ops.history_gram``), so agents that keep pushing the model the same way lose their weight.
``--aggr flare`` weights that launch by FLARE's trust: the MMD between the participants' penultimate-layer representations of a clean
root set (``ops.flare_sums`` on the features the engine computes) and a softmax over how often each is among the others' nearest
neighbours (``ops.flare_weights``).
``--aggr deepsight`` runs that launch with equal weights over DeepSight's accepted clusters, clipped to the median norm: the statistics
of the participants' output layers and of their behaviour on random inputs (``ops.deepsight_stats`` on the logits the engine computes)
label and cluster them (``ops.deepsight_decide``).
``--detect fldetector`` is a stage ahead of the rule: every round it predicts each agent's update from its last one and an L-BFGS
Hessian-vector product of the recent global updates (``ops.fld_hvp_coefficients`` on the Gram matrix of the update ring,
``ops.fld_hvp``), scores the distance to the prediction (``ops.fld_predict``) and, once the gap statistic finds a minority cluster of high
scores (``ops.fld_detect``), removes those agents from every later round's admission.
The reference's dead / disabled pieces are available behind flags: ``clip_updates`` (``--server_clip``) and the
diagnostics ``plot_norms`` / ``comp_diag_fisher`` / ``plot_sign_agreement`` (``--diagnostics``), the latter with the
reference's latent bugs fixed (model built on the right device; Fisher uses log-probabilities -- SURVEY.md quirk 7).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import ops
from .models.graph import GraphNet, head_slices


def server_opt_spec(args):
    """``ops.ServerOptState`` keyword arguments of the ``--server_opt*`` flags."""
    return dict(kind=getattr(args, "server_opt", "sgd"), beta1=getattr(args, "server_beta1", 0.9),
                beta2=getattr(args, "server_beta2", 0.99), tau=getattr(args, "server_tau", 1e-3))


# TensorBoard tags of FLDetector's record fields (a list of flagged ids is logged as its length)
_FLD_TAGS = {"fld_avg_honest_score": "FLDetector/Avg_Honest_Score", "fld_avg_corrupt_score": "FLDetector/Avg_Corrupt_Score",
             "fld_clusters": "FLDetector/Clusters", "fld_fallback": "FLDetector/Fallback", "fld_flagged": "FLDetector/Flagged",
             "fld_corrupt_flagged": "FLDetector/Corrupt_Flagged", "fld_excluded": "FLDetector/Excluded"}


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
        self.last_foolsgold = None    # the FoolsGold/* scalars of the last round (--aggr foolsgold)
        self.last_flare = None        # the FLARE/* scalars of the last round (--aggr flare)
        self.last_deepsight = None    # the DeepSight/* scalars of the last round (--aggr deepsight)
        self.history = None           # [num_agents][n_vote] FoolsGold histories of the in-process form (allocated on first use)
        self.opt = None               # full-length server optimizer state of the in-process form (allocated on first use)
        # FLDetector (--detect fldetector): host state identical on every rank, and the in-process form's tables (allocated on first use)
        self.last_fld = None          # the fld_* record fields of the last round
        self.fld_count = 0            # valid ring rows (at most N + 1)
        self.fld_pos = 0              # the ring row the next global update goes to (the oldest one once the ring is full)
        self.fld_window = []          # the last N round scores, oldest first: float64 [num_agents] each
        self.fld_flagged = []         # agent ids flagged at detection (ascending)
        self.fld_detect_round = None  # the round of the detection, None until then
        self.fld_tables = None        # (table [num_agents][n_vote], ring [N + 1][n_vote], w_prev [n_vote]) of the in-process form
        # SparseFed (--server_topk) of the in-process form: the error vector [n_vote] (allocated on first use) and the last round's fields
        self.sparse_e = None
        self.last_sparse = None
        # CRFL (--param_clip / --param_noise) of the in-process form: the real-coordinate mask (built on first use) and the last round's fields
        self.crfl_mask = None
        self.last_crfl = None

    # ---- the server step ------------------------------------------------------------------------------------
    def aggregate_updates(self, w_global, agent_params, cur_round, n_vote=None, root_params=None, features=None, logits=None,
                          global_logits=None):
        """In-process form: ``agent_params`` = {agent_id: flat local parameters}.  Updates ``w_global`` in place.  ``root_params``:
        the server's root-trained parameters, needed by ``--aggr fltrust``; ``features``: fp32 ``[K][n][d]`` root-set features of the
        participants in ``agent_params``' order, needed by ``--aggr flare``; ``logits`` / ``global_logits``: fp32 ``[K][S N][P]`` logits
        of those participants and ``[S N][P]`` of ``w_global`` on DeepSight's random inputs, needed by ``--aggr deepsight``."""
        ids = list(agent_params.keys())
        ws = [agent_params[i] for i in ids]
        nv = n_vote if n_vote is not None else (self.layout.n_vote if self.layout else None)
        if self._fltrust and root_params is None:
            raise ValueError("--aggr fltrust needs the server's root parameters (root_params)")
        if self._flare and features is None:
            raise ValueError("--aggr flare needs the participants' root-set features (features)")
        if self._deepsight and (logits is None or global_logits is None):
            raise ValueError("--aggr deepsight needs the participants' and the global model's logits (logits, global_logits)")
        clip = self._clip_scales(ops.update_norms(w_global, ws, nv)) if self._server_clip else None
        all_ids, all_ws = ids, ws
        n_voted = nv if nv is not None else w_global.numel()
        distances = lambda: ops.pairwise_sqdist(ws, n_voted, w_global if clip is not None else None, clip)
        dnc = lambda: ops.dnc_grams(ws, w_global, self._dnc_samples(cur_round, n_voted), n_voted, clip)
        rfa_pass = lambda b, members: ops.rfa_sqdist(
            [ws[j] for j in members], b, nv, w_global if clip is not None else None,
            clip[torch.as_tensor(members, device=clip.device)] if clip is not None else None)
        gram = lambda members: ops.pairwise_gram([ws[j] for j in members], w_global, nv)
        detection = lambda: self._fld_stage(ids, cur_round, *self._fld_local(w_global, ws, ids, nv))
        keep, weights, scales, total, noise_std = self._admission(ids, clip, detection, distances, dnc,
                                                                  lambda: ops.trust_stats(ws, root_params, w_global, nv), rfa_pass, gram,
                                                                  lambda members: self._history_pass(w_global, ws, ids, members, nv),
                                                                  cur_round, lambda: features,
                                                                  lambda: (ops.deepsight_stats(logits, global_logits, ws, w_global,
                                                                                               head_slices(self.layout)),
                                                                           ops.update_norms(w_global, ws, nv)))
        if keep is not None and len(keep) < len(ids):
            ids, ws, weights = [ids[j] for j in keep], [ws[j] for j in keep], [weights[j] for j in keep]
            scales = scales[torch.as_tensor(keep, device=scales.device)] if scales is not None else None
        prev = w_global.clone() if self.args.diagnostics else None
        flipped = torch.zeros(1, dtype=torch.int64, device=w_global.device)
        if self.opt is None:
            self.opt = ops.ServerOptState(n=w_global.numel(), device=w_global.device, **server_opt_spec(self.args))
        p = float(getattr(self.args, "server_topk", 0.0))
        rho, sigma = float(getattr(self.args, "param_clip", 0.0)), float(getattr(self.args, "param_noise", 0.0))
        crfl = rho > 0 or sigma > 0
        # SparseFed / CRFL: the plain step's result w' goes to a scratch vector
        out = torch.empty_like(w_global) if (p > 0 or crfl) else w_global
        ops.fused_aggregate(w_global, ws, weights, self._mode, self.args.robustLR_threshold, self.server_lr, noise_std, self.args.seed,
                            cur_round,
                            n_vote if n_vote is not None else (self.layout.n_vote if self.layout else None),
                            scales, out=out, flipped=flipped, opt=self.opt, total_weight=total)
        if p > 0:
            k = ops.sparsefed_k(p, self.n_params)
            if self.sparse_e is None:
                self.sparse_e = torch.zeros(n_voted, dtype=torch.float32, device=w_global.device)
            stats = torch.zeros(3, dtype=torch.float64, device=w_global.device)
            ops.sparsefed_step(w_global, out, self.sparse_e, n_voted, k, stats)
            s = stats.tolist()
            self.last_sparse = {"sparse_applied": int(s[0]), "sparse_threshold": s[1], "sparse_error_norm": s[2]}
            out = w_global                                            # CRFL's pass follows in place
        if crfl:
            if self.layout is None:
                raise ValueError("--param_clip / --param_noise need the model's layout (its real-coordinate mask)")
            if self.crfl_mask is None:
                self.crfl_mask = ops.real_mask(self.layout).to(w_global.device)
            stats = torch.zeros(2, dtype=torch.float64, device=w_global.device)
            ops.crfl_step(w_global, out, self.crfl_mask, self.layout.n_vote, rho, sigma, self.args.seed, cur_round, stats)
            s = stats.tolist()
            self.last_crfl = {"param_norm": s[0], "param_scale": s[1]}
        self.last_flipped = flipped
        if self.args.diagnostics:
            self.plot_norms(dict(zip(all_ids, ops.update_norms(prev, all_ws, nv).tolist())), cur_round)
            self.plot_sign_agreement(prev, w_global, ws, ids, cur_round)     # the vote that happened: admitted participants only
        return

    def aggregate_slots(self, participants, cur_round, flare_local=None, deepsight_local=None):
        """Engine form: participant j's parameters live in ``fused.slot_owner(j)``; updates every rank's global.  Under
        ``--aggr fltrust`` the server's root job is position ``len(participants)``.  ``flare_local``: under ``--aggr flare``, this rank's
        ``[max_slots][n][d]`` root-set features of the participants in its slots (``FusedAggregator.flare_features``).
        ``deepsight_local``: under ``--aggr deepsight``, this rank's ``[max_slots][(S + 2) P]`` DeepSight statistics of the participants
        in its slots (``ops.deepsight_stats``), all-gathered the same way."""
        K = len(participants)
        diag = bool(self.args.diagnostics)
        norms = self.fused.update_norms(K) if self._server_clip or diag else None
        clip = self._clip_scales(norms) if self._server_clip else None
        copies, gathered = None, None
        if (self._selecting or self._fltrust or self._flame or self._foolsgold or self._detecting or (self._rfa and self.args.rfa_iters > 0)) \
                and self.fused.gathers(K):
            # on the gather transport every pass reads the same all-gathered copies (one all_gather per round; the root job included)
            gathered = self.fused.gather_participants(K + 1 if self._fltrust else K)
            copies = gathered[:K]
        fused = self.fused
        detection = lambda: self._fld_stage(participants, cur_round, fused.fld_ring_update, fused.fld_gram,
                                            lambda order, coef: fused.fld_predict(K, participants, order, coef, copies))
        keep, weights, scales, total, noise_std = self._admission(
            participants, clip, detection, lambda: self.fused.pairwise_sqdist(K, clip, copies),
            lambda: self.fused.dnc_grams(K, self._dnc_samples(cur_round, self.fused.n_vote), clip, None, copies),
            lambda: self.fused.trust_stats(K, K, gathered),
            lambda b, members: self.fused.rfa_sqdist(K, b, clip, members, copies),
            lambda members: self.fused.pairwise_gram(K, members, copies),
            lambda members: self.fused.foolsgold_gram(K, participants, members, copies), cur_round,
            lambda: self.fused.flare_features(K, flare_local),
            lambda: (self.fused.gather_slot_rows(K, deepsight_local), norms if norms is not None else self.fused.update_norms(K)))
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

    def _admission(self, ids, clip, detection, distances, dnc_grams, trust_stats, rfa_pass, gram, history, cur_round, features=None,
                   deepsight=None):
        """Admission of the participants ``ids`` shared by both forms of the step: FLDetector's ``detection()`` (``--detect``), which returns
        the positions of the agents it has not flagged (None while it has flagged nobody), or Krum / Multi-Krum on ``distances()`` or DnC
        on its Gram matrices ``dnc_grams()`` (``--select``),
        then FLTrust on ``trust_stats()`` (``--aggr fltrust``), RFA's weights from ``rfa_pass(b, members)`` (``--aggr rfa``), FLAME on
        the Gram matrix ``gram(members)`` (``--aggr flame``) or FoolsGold on ``history(members)``, the Gram matrix of the members' update
        histories after this round's updates are folded in (``--aggr foolsgold``), or FLARE on the participants' root-set features
        ``features()`` (``--aggr flare``), or DeepSight on ``deepsight()``, the participants' statistics and update norms (``--aggr
        deepsight``).  ``clip``: the server-clipping scales or None.  Returns
        ``(members, weights, scales, total_weight, noise_std)`` for the step: members None admits everyone; weights are per position in
        ``ids``."""
        keep = self._admit(ids, cur_round, distances, dnc_grams) if self._select else (detection() if self._detect else None)
        noise_std = self.args.noise * self.args.clip
        if self._fltrust:
            return (*self._trust(trust_stats(), ids, keep, cur_round), noise_std)
        if self._flame:
            return self._flame_step(ids, keep, gram, cur_round)
        if self._flare:
            members, weights, total = self._flare_step(ids, keep, features, cur_round)
            return members, weights, clip, total, noise_std
        if self._deepsight:
            return (*self._deepsight_step(ids, keep, deepsight, cur_round), noise_std)
        weights = [float(self.agent_data_sizes[i]) for i in ids]
        if self._foolsgold:
            members, weights, total = self._foolsgold_step(ids, keep, weights, history, cur_round)
            return members, weights, clip, total, noise_std
        if self._rfa:
            return (*self._rfa_weights(ids, keep, weights, clip, rfa_pass, cur_round), noise_std)
        return keep, weights, clip, None, noise_std

    @property
    def _detect(self):
        return getattr(self.args, "detect", "none") == "fldetector"

    @property
    def _detecting(self):
        """True while the FLDetector pass runs: from the first round until the detection."""
        return self._detect and self.fld_detect_round is None

    def _fld_local(self, w_global, ws, ids, nv):
        """The ring, Gram and prediction passes of the in-process form, on full tables kept here (zero at the start)."""
        nv = w_global.numel() if nv is None else int(nv)
        if self.fld_tables is None:
            z = lambda *shape: torch.zeros(shape, dtype=torch.float32, device=w_global.device)
            self.fld_tables = (z(self.args.num_agents, nv), z(self.args.fld_window + 1, nv), z(nv))
        table, ring, w_prev = self.fld_tables

        def predict(order, coef):
            hv = ops.fld_hvp([ring[i] for i in order], coef, 0, nv) if coef is not None else None
            return ops.fld_predict([table[i] for i in ids], ws, w_global, hv, 0, nv)
        return (lambda row: ops.fld_ring(w_global, w_prev, None if row is None else ring[row], 0, nv),
                lambda order: ops.history_gram([ring[i] for i in order], nv), predict)

    def _fld_stage(self, ids, cur_round, ring, gram, predict):
        """FLDetector ahead of the rule (DESIGN.md section 3), over the participants ``ids`` (every agent: all take part in every round).
        Until the detection: ``ring(row)`` writes the round's global update into ring row ``row`` (None in round 1: only w_prev), from round
        N + 2 on ``gram(order)`` gives the ring's Gram matrix, ``ops.fld_hvp_coefficients`` the Hessian-vector product and ``predict(order,
        coef)`` the squared distances to the predictions (``predict(None, None)`` before: record only); the round scores enter the window
        and from round max(R, 2N + 1) on ``ops.fld_detect`` decides.  Returns the positions of the agents not flagged, or None while nobody
        is flagged.  Records ``last_fld`` and logs it."""
        a = self.args
        N, nc = a.fld_window, a.num_corrupt
        rec = {}
        if self.fld_detect_round is None:
            if cur_round >= 2:
                ring(self.fld_pos)
                self.fld_pos = (self.fld_pos + 1) % (N + 1)
                self.fld_count = min(N + 1, self.fld_count + 1)
            else:
                ring(None)
            if cur_round >= N + 2:
                if self.fld_count != N + 1:
                    raise ValueError(f"FLDetector: round {cur_round} with {self.fld_count} of {N + 1} ring rows")
                order = [(self.fld_pos + i) % (N + 1) for i in range(N + 1)]       # oldest first: pos is the next row to overwrite
                coef = ops.fld_hvp_coefficients(gram(order))
                d = np.sqrt(np.maximum(predict(order, coef).double().cpu().numpy(), 0.0))
                tot = float(d.sum())
                score = np.zeros(a.num_agents, dtype=np.float64)
                score[np.asarray(ids, dtype=np.int64)] = d / tot if tot > 0 else 0.0
                self.fld_window = (self.fld_window + [score])[-N:]
                rec["fld_fallback"] = int(not np.any(coef))
            else:
                predict(None, None)
            if len(self.fld_window) == N:
                sus = self.fld_window[0].copy()
                for w in self.fld_window[1:]:
                    sus = sus + w
                sus = sus / N
                cand = sorted(int(i) for i in ids)
                honest, corrupt = [sus[i] for i in cand if i >= nc], [sus[i] for i in cand if i < nc]
                rec["fld_avg_honest_score"] = float(np.mean(honest)) if honest else None
                rec["fld_avg_corrupt_score"] = float(np.mean(corrupt)) if corrupt else None
                if cur_round >= max(a.fld_start, 2 * N + 1):
                    flagged, khat = ops.fld_detect(sus[cand], a.seed, cur_round)
                    rec["fld_clusters"] = khat
                    if flagged:
                        self.fld_flagged = [cand[j] for j in flagged]
                        self.fld_detect_round = cur_round
                        rec["fld_flagged"] = list(self.fld_flagged)
                        rec["fld_corrupt_flagged"] = sum(1 for i in self.fld_flagged if i < nc)
                        rec["fld_detect_round"] = cur_round
        keep = None
        if self.fld_flagged:
            out = set(self.fld_flagged)
            keep = [j for j, i in enumerate(ids) if int(i) not in out]
            rec["fld_excluded"] = len(ids) - len(keep)
        self.last_fld = rec
        if self.writer is not None:
            for k, v in rec.items():
                if k in _FLD_TAGS and v is not None:
                    self.writer.add_scalar(_FLD_TAGS[k], len(v) if isinstance(v, list) else v, cur_round)
        return keep

    def fld_state(self):
        """FLDetector's host state, as a checkpoint carries it."""
        return {"count": self.fld_count, "pos": self.fld_pos, "window": [torch.from_numpy(w.copy()) for w in self.fld_window],
                "flagged": list(self.fld_flagged), "detect_round": self.fld_detect_round}

    def load_fld_state(self, st):
        self.fld_count, self.fld_pos = int(st["count"]), int(st["pos"])
        self.fld_window = [w.double().numpy().copy() for w in st["window"]]
        self.fld_flagged = [int(i) for i in st["flagged"]]
        self.fld_detect_round = st["detect_round"]

    def _admit(self, ids, cur_round, distances, dnc_grams):
        """``--select`` admission of the participants ``ids``: Krum / Multi-Krum from the pairwise distances ``distances()``, or DnC from
        the Gram matrices ``dnc_grams()`` of this round's subsamples (everyone, with nothing launched, when it removes ``floor(c F) = 0``).
        Returns the admitted positions (ascending).  Records ``last_admitted`` and logs how many corrupt participants (ids < num_corrupt)
        came and got through."""
        a = self.args
        if a.select != "dnc":
            keep = ops.krum_select(distances(), ids, a.select_f, a.select_m)
        elif self._selecting:
            keep = ops.dnc_select(dnc_grams(), ids, a.select_f, a.dnc_frac)
        else:
            keep = list(range(len(ids)))
        self.last_admitted = [ids[j] for j in keep]
        nc = self.args.num_corrupt
        self.last_select = {"Select/Corrupt_Participants": sum(1 for i in ids if i < nc),
                            "Select/Corrupt_Admitted": sum(1 for i in self.last_admitted if i < nc)}
        if self.writer is not None:
            for k, v in self.last_select.items():
                self.writer.add_scalar(k, v, cur_round)
        return keep

    @property
    def _selecting(self):
        """True when ``--select`` runs a device pass this round: always for krum / multikrum, for dnc unless it removes nobody."""
        if getattr(self.args, "select", "none") == "dnc":
            return math.floor(self.args.dnc_frac * self.args.select_f) > 0
        return self._select

    def _dnc_samples(self, cur_round, n_vote):
        """This round's DnC subsamples: ``ops.dnc_sample`` of every iteration, int64 numpy ``[T][min(b, n_vote)]``."""
        a = self.args
        return np.stack([ops.dnc_sample(a.seed, cur_round, t, a.dnc_dim, n_vote) for t in range(a.dnc_iters)])

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
    def _foolsgold(self):
        return self.args.aggr == "foolsgold"

    @property
    def _flare(self):
        return self.args.aggr == "flare"

    @property
    def _deepsight(self):
        return self.args.aggr == "deepsight"

    @property
    def _mode(self):
        """The aggregate kernel's rule: FLTrust is its weighted mean with trust weights and per-participant scales, RFA with its
        Weiszfeld weights, FLAME with equal weights and its clip scales, FoolsGold with its weights times the data sizes, FLARE with its
        trust scores, DeepSight with equal weights and its clip scales."""
        return "avg" if self._fltrust or self._rfa or self._flame or self._foolsgold or self._flare or self._deepsight else self.args.aggr

    def _history_pass(self, w_global, ws, ids, members, nv):
        """In-process form of the FoolsGold history pass: fold the updates of the participants at positions ``members`` into the rows of
        their agents in ``self.history`` (a full-length ``[num_agents][n_vote]`` table on ``w_global``'s device, zero at the start) and
        return the Gram matrix of those rows."""
        nv = w_global.numel() if nv is None else int(nv)
        if self.history is None:
            self.history = torch.zeros((self.args.num_agents, nv), dtype=torch.float32, device=w_global.device)
        rows = [self.history[ids[j]] for j in members]
        ops.history_accumulate(rows, [ws[j] for j in members], w_global, 0, nv)
        return ops.history_gram(rows, nv)

    def _foolsgold_step(self, ids, keep, weights, history, cur_round):
        """FoolsGold over the positions ``keep`` that selection admitted (all when None): ``ops.foolsgold_weights`` on ``history(candidates)``.
        Returns ``(members, weights, total_weight)`` for the step: the candidates with alpha > 0, weights alpha times the data sizes
        ``weights`` and total weight their sum -- or, when every alpha is 0, every candidate with weight 0 and total weight 1, so the
        aggregate is 0 plus noise.  A round in which every alpha is 1 is the avg step bit for bit.  Records ``last_admitted`` and logs the
        mean alpha of honest (ids >= num_corrupt) and corrupt candidates and the admitted count."""
        K = len(ids)
        cand = list(range(K)) if keep is None else [int(j) for j in keep]
        alpha = ops.foolsgold_weights(history(cand))
        members = [j for j, a in zip(cand, alpha) if a > 0]
        w = [0.0] * K
        for j, a in zip(cand, alpha):
            w[j] = float(a) * weights[j]
        total = sum(w[j] for j in members)
        self.last_admitted = [ids[j] for j in members]
        if not members:
            members, w, total = cand, [0.0] * K, 1.0
        nc = self.args.num_corrupt
        honest = [float(a) for j, a in zip(cand, alpha) if ids[j] >= nc]
        corrupt = [float(a) for j, a in zip(cand, alpha) if ids[j] < nc]
        self.last_foolsgold = {"FoolsGold/Avg_Honest_Weight": sum(honest) / len(honest) if honest else None,
                               "FoolsGold/Avg_Corrupt_Weight": sum(corrupt) / len(corrupt) if corrupt else None,
                               "FoolsGold/Admitted": len(self.last_admitted)}
        if self.writer is not None:
            for k, v in self.last_foolsgold.items():
                if v is not None:
                    self.writer.add_scalar(k, v, cur_round)
        return members, w, total

    def _flare_step(self, ids, keep, features, cur_round):
        """FLARE over the positions ``keep`` that selection or detection admitted (all when None): ``ops.flare`` on the candidates' rows of
        ``features()`` (fp32 ``[K][n][d]``, identical on every rank).  Returns ``(members, weights, total_weight)`` for the step: F, the
        candidates whose features are all finite, with weights ``fp32(TS_j)`` and total weight the sum of those fp32 weights (data sizes
        are not used) -- or, when F is empty, every candidate with weight 0 and total weight 1, so the aggregate is 0 plus noise.  Records
        ``last_admitted`` (F) and logs the mean trust of honest (ids >= num_corrupt) and corrupt candidates, the corrupt share of the
        trust and the bandwidth sigma^2."""
        K = len(ids)
        cand = list(range(K)) if keep is None else [int(j) for j in keep]
        Z = features()
        if cand != list(range(K)):
            Z = Z[torch.as_tensor(cand, dtype=torch.int64, device=Z.device)]
        res = ops.flare(Z, self.args.flare_k, self.args.flare_tau)
        members = [cand[j] for j in res.members]
        w = [0.0] * K
        for j, t in zip(cand, res.weights):
            w[j] = float(np.float32(t))
        total = sum(w[j] for j in members)
        self.last_admitted = [ids[j] for j in members]
        if not members:
            members, w, total = cand, [0.0] * K, 1.0
        nc = self.args.num_corrupt
        honest = [float(t) for j, t in zip(cand, res.weights) if ids[j] >= nc]
        corrupt = [float(t) for j, t in zip(cand, res.weights) if ids[j] < nc]
        self.last_flare = {"FLARE/Avg_Honest_Trust": sum(honest) / len(honest) if honest else None,
                           "FLARE/Avg_Corrupt_Trust": sum(corrupt) / len(corrupt) if corrupt else None,
                           "FLARE/Corrupt_Weight": sum(corrupt), "FLARE/Bandwidth": res.sigma2}
        if self.writer is not None:
            for k, v in self.last_flare.items():
                if v is not None:
                    self.writer.add_scalar(k, v, cur_round)
        return members, w, total

    def _deepsight_step(self, ids, keep, deepsight, cur_round):
        """DeepSight over the positions ``keep`` that selection or detection admitted (all when None): ``ops.deepsight_decide`` on the
        candidates' rows of ``deepsight()`` = (statistics ``[K][(S + 2) P]``, update norms ``[K]``), identical on every rank.  Returns
        ``(members, weights, scales, total_weight)`` for the step: the accepted positions with weight 1 each, total weight their count
        and the clip scales -- or, when nobody is accepted, every candidate with weight 0 and total weight 1, so the aggregate is 0 plus
        noise.  Records ``last_admitted`` and logs the accepted and suspicious counts, the corrupt ones among them (ids < num_corrupt),
        the number of final clusters over the finite candidates and the clip bound."""
        K = len(ids)
        cand = list(range(K)) if keep is None else [int(j) for j in keep]
        stats, norms = deepsight()
        idx = torch.as_tensor(cand, dtype=torch.int64)
        res = ops.deepsight_decide(stats.detach().cpu()[idx], norms.detach().double().cpu()[idx], [ids[j] for j in cand],
                                   self.args.deepsight_tau)
        members = [cand[j] for j in res.members]
        scales = torch.ones(K, dtype=torch.float32)
        scales[idx] = res.scales
        weights, total = [1.0] * K, float(len(members))
        self.last_admitted = [ids[j] for j in members]
        if not members:
            members, weights, total = cand, [0.0] * K, 1.0
        nc = self.args.num_corrupt
        sus = [ids[cand[j]] for j in range(len(cand)) if res.suspicious[j]]
        self.last_deepsight = {"DeepSight/Accepted": len(self.last_admitted),
                               "DeepSight/Corrupt_Accepted": sum(1 for i in self.last_admitted if i < nc),
                               "DeepSight/Suspicious": len(sus), "DeepSight/Corrupt_Suspicious": sum(1 for i in sus if i < nc),
                               "DeepSight/Clusters": len({int(v) for v in res.labels if v >= 0}),
                               "DeepSight/Clip_Bound": res.clip_bound}
        if self.writer is not None:
            for k, v in self.last_deepsight.items():
                if v is not None:
                    self.writer.add_scalar(k, v, cur_round)
        return members, weights, scales, total

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
