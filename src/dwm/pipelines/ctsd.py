"""CTSD inference pipelines — mirror of the inference part of reference
src/dwm/pipelines/ctsd.py: `CrossviewTemporalSD` (ctor :844-1012, condition building
:84-464, `inference_pipeline` :1439-1654, `autoregressive_inference_pipeline` :1656-1833)
and `StreamingCrossviewTemporalSD` (diffusion-forcing FIFO :2010-2277).

Scope (SURVEY.md §8): the denoise loop, its integer timestep-index schedule, CFG
batching, the model call and the scheduler update run on the H100-native kernels
(`model.forward_tokens` + one fused CFG / un-patchify / per-frame-Euler / masked-update
kernel per step, no host synchronisation inside the loop); the VAE decode runs on the
mirrored CogVideoX / AutoencoderKL decoders (loaded from `<path>/vae`, or supplied as
`common_config["vae_instance"]`; without one the exiting latents are returned).
Training, evaluation and preview dumping are not mirrored.  Text conditions come from the
batch's `clip_text` prompts through Hugging Face CLIP / T5 when the checkpoint directory
holds the encoders (`dwm.pipelines.text_conditions`, a caller of the hot path), or
pre-encoded (`text_embeddings` / `pooled_text_embeddings` and their `uncond_*` twins for
classifier-free guidance).

The host logic is held to the reference's own code by `tests/test_reference_golden.py`
(condition tensors, loop outputs and orchestration call traces recorded from
/root/reference/src on a `diffusers` name shim).
"""
import os

import torch

import dwm.common
import dwm.functional
from dwm import _compat
from dwm.schedulers import temporal_independent as _ti
from opendwm_b200 import ops as _ops


def load_vae(vae_type, vae_path, common_config):
    """vae_type.from_pretrained(vae_path, subfolder="vae"), with common_config["vae_gemm_dtype"]
    (a dtype, or its {"_class_name": "get_class", "class_name": ...} config) as the opt-in
    gemm_dtype of the decoder ResNet convolutions."""
    gemm_dtype = dwm.common.create_instance_from_config(common_config.get("vae_gemm_dtype"))
    kw = {} if gemm_dtype is None else {"gemm_dtype": gemm_dtype}
    return vae_type.from_pretrained(vae_path, subfolder="vae", **kw)


class CrossviewTemporalSD:

    @staticmethod
    def load_state(path: str):
        """reference :29-36."""
        if path.endswith(".safetensors"):
            import safetensors.torch
            return safetensors.torch.load_file(path, device="cpu")
        return torch.load(path, map_location="cpu", weights_only=True)

    @staticmethod
    def get_camera_transform_ids(batch, common_config):
        """reference :84-95."""
        return torch.cat([
            batch["camera_intrinsics"].flatten(-2, -1)[
                ..., common_config["camera_intrinsic_embedding_indices"]
            ] / batch["image_size"][
                ..., common_config["camera_intrinsic_denom_embedding_indices"]
            ],
            batch["camera_transforms"].flatten(-2, -1)[
                ..., common_config["camera_transform_embedding_indices"]
            ]
        ], -1)

    @staticmethod
    def get_action_ids(batch, common_config: dict, action_condition_mask=None,
                       streaming_mode: bool = False, prev_ego_transforms=None):
        """Speed (km/h) and steering from consecutive ego poses; -1000 marks the
        unconditional case (reference :97-156)."""
        if streaming_mode:
            assert batch["ego_transforms"].shape[1] == 1
            ego_transforms = torch.cat([
                batch["ego_transforms"] if prev_ego_transforms is None
                else prev_ego_transforms,
                batch["ego_transforms"]], dim=1)
        else:
            ego_transforms = batch["ego_transforms"]
        current_pose = ego_transforms[
            :, :, common_config["camera_ego_sensor_indices"]]
        uncondition_pose = torch.eye(4).view(1, 1, 1, 4, 4)
        is_conditioned = (current_pose - uncondition_pose)\
            .sum((1, 2, 3, 4)).abs() > 1e-3
        if action_condition_mask is not None:
            is_conditioned = torch.logical_and(
                is_conditioned, action_condition_mask)
        relative_pose = torch.linalg.solve(
            current_pose[:, :-1], current_pose[:, 1:])
        relative_pose = torch.cat([relative_pose[:, :1], relative_pose], 1)
        moving_distance = torch.norm(
            relative_pose[..., :3, 3], dim=-1, keepdim=True)
        speed = 3.6 * moving_distance * batch["fps"].view(-1, 1, 1, 1)
        rotation_angles = torch.atan2(
            relative_pose[..., 1, 0:1] - relative_pose[..., 0, 1:2],
            relative_pose[..., 0, 0:1] + relative_pose[..., 1, 1:2])
        wheel_base, steering_ratio = 2.7, 14
        steering = torch.where(
            torch.abs(moving_distance) > 0.01,
            rotation_angles / moving_distance * wheel_base * steering_ratio,
            -1000.0 * torch.ones_like(rotation_angles))
        action_ids = torch.cat([speed, steering], -1)
        action_ids = torch.where(
            is_conditioned.view(-1, 1, 1, 1), action_ids,
            -1000.0 * torch.ones_like(action_ids))
        if streaming_mode:
            action_ids = action_ids.chunk(2, dim=1)[-1]
        return action_ids

    @staticmethod
    def get_conditions(model, text_encoder, tokenizer, common_config: dict,
                       latent_shape, batch: dict, device, dtype,
                       text_condition_mask=None, _3dbox_condition_mask=None,
                       hdmap_condition_mask=None, action_condition_mask=None,
                       explicit_view_modeling_mask=None,
                       streaming_mode: bool = False, prev_ego_transforms=None,
                       do_classifier_free_guidance: bool = False,
                       latents_shape=None):
        """Model kwargs from a data batch (reference :158-464).  Text: a batch with
        pre-encoded `text_embeddings` [B,T,V,L,C] / `pooled_text_embeddings` [B,T,V,P] uses
        them (uncond half = `uncond_*` entries, or zeros when absent; `text_encoder` then only
        needs to be not None); a batch with `clip_text` prompts goes through the given
        encoders / tokenizers like the reference does."""
        batch_size, _, view_count = latent_shape[:3]
        sequence_length = batch["pts"].shape[1]
        if do_classifier_free_guidance:
            batch_size *= 2
        if common_config.get("explicit_view_modeling", False):
            raise NotImplementedError(
                "explicit_view_modeling (UniMLVG) is outside the CTSD hot path")

        encoder_hidden_states = pooled = None
        if text_encoder is not None and "text_embeddings" in batch:
            te = batch["text_embeddings"].to(device=device, dtype=dtype)
            pe = batch["pooled_text_embeddings"].to(device=device, dtype=dtype)
            if do_classifier_free_guidance:
                ute = batch.get("uncond_text_embeddings", torch.zeros_like(te))\
                    .to(device=device, dtype=dtype)
                upe = batch.get("uncond_pooled_text_embeddings",
                                torch.zeros_like(pe)).to(device=device, dtype=dtype)
                te, pe = torch.cat([ute, te]), torch.cat([upe, pe])
            encoder_hidden_states, pooled = te, pe
        elif text_encoder is not None and "clip_text" in batch:
            # reference-style prompts through the real text encoders (reference :176-253)
            if isinstance(text_encoder, str):
                raise RuntimeError(
                    "the batch carries prompts (clip_text) but no text encoders were loaded: "
                    "point pretrained_model_name_or_path at a checkpoint directory with "
                    "tokenizer*/text_encoder* or pass pre-encoded text_embeddings")
            from dwm.pipelines.text_conditions import text_conditions
            encoder_hidden_states, pooled = text_conditions(
                isinstance(model, _compat.SD3Transformer2DModelMarker), text_encoder, tokenizer,
                batch["clip_text"], sequence_length, view_count, device, dtype,
                text_condition_mask, do_classifier_free_guidance)

        condition_on_all_frames = common_config.get(
            "condition_on_all_frames", False)
        color = common_config.get("uncondition_image_color", 0)
        condition_image_list = []
        for key, mask in (("3dbox_images", _3dbox_condition_mask),
                          ("hdmap_images", hdmap_condition_mask)):
            if key not in batch:
                continue
            img = batch[key].to(device) if condition_on_all_frames \
                else batch[key][:, :1].to(device)
            if mask is not None:
                img = img.clone()
                img[mask.logical_not().to(device)] = color
            if do_classifier_free_guidance:
                img = torch.cat([torch.ones_like(img) * color, img])
            condition_image_list.append(img)
        condition_image_tensor = torch.cat(condition_image_list, -3) \
            if condition_image_list else None

        added_time_ids = None
        kind = common_config.get("added_time_ids")
        if kind in ("fps_camera_transforms", "fps_camera_transforms_action"):
            parts = [
                batch["fps"].view(-1, 1, 1, 1)
                .repeat(1, sequence_length, view_count, 1),
                CrossviewTemporalSD.get_camera_transform_ids(batch, common_config)]
            if kind == "fps_camera_transforms_action":
                parts.append(CrossviewTemporalSD.get_action_ids(
                    batch, common_config, action_condition_mask,
                    streaming_mode, prev_ego_transforms))
            added_time_ids = torch.cat(parts, -1)
            if do_classifier_free_guidance:
                if kind == "fps_camera_transforms_action":
                    uncond = torch.cat([
                        added_time_ids[..., :-2],
                        -1000 * torch.ones_like(added_time_ids[..., -2:])], -1)
                else:
                    uncond = added_time_ids
                added_time_ids = torch.cat([uncond, added_time_ids], 0)
            added_time_ids = added_time_ids.to(device)

        has_depth_input = "camera_intrinsics" in batch and \
            "camera_transforms" in batch
        rep = (lambda t: torch.cat([t, t])) if do_classifier_free_guidance \
            else (lambda t: t)
        result = {
            "encoder_hidden_states": encoder_hidden_states,
            "condition_image_tensor": condition_image_tensor,
            "disable_crossview": torch.tensor(
                [common_config.get("disable_crossview", False)],
                device=device).repeat(batch_size),
            "disable_temporal": torch.tensor(
                [common_config.get("disable_temporal", False)],
                device=device).repeat(batch_size),
            "crossview_attention_mask":
                rep(batch["crossview_mask"]).to(device)
                if "crossview_mask" in batch else None,
            "camera_intrinsics": rep(batch["camera_intrinsics"].to(device))
                if has_depth_input else None,
            "camera_transforms": rep(batch["camera_transforms"].to(device))
                if has_depth_input else None,
            "camera_intrinsics_norm": None,
            "camera2referego": None,
            "added_time_ids": added_time_ids,
        }
        if isinstance(model, _compat.SD3Transformer2DModelMarker) and \
                text_encoder is not None:
            result["pooled_projections"] = pooled

        if latents_shape is not None and latents_shape[1] != sequence_length:
            pre = 1 if sequence_length % 2 == 1 else 0
            stride = (sequence_length - pre) // (latents_shape[1] - pre)
            for k in result:
                if result[k] is not None and result[k].ndim > 1 and \
                        result[k].shape[1] == sequence_length:
                    result[k] = torch.cat(
                        [result[k][:, :pre], result[k][:, pre::stride]], dim=1)
        return result

    def __init__(self, output_path, config: dict, device, common_config: dict,
                 training_config: dict, inference_config: dict,
                 pretrained_model_name_or_path: str, model, model_dtype=None,
                 model_checkpoint_path=None, model_load_state_args: dict = {},
                 metrics: dict = {}, resume_from=None):
        self.should_save = not torch.distributed.is_initialized() or \
            torch.distributed.get_rank() == 0
        self.config = config
        self.device = torch.device(device)
        self.common_config = common_config
        self.training_config = training_config
        self.inference_config = inference_config
        self.output_path = output_path
        if self.device.type != "cuda":
            raise RuntimeError(
                "dwm.pipelines.ctsd runs on CUDA (sm_90a) only; there is no CPU "
                "fallback")

        self.generator = torch.Generator()
        if "generator_seed" in self.config:
            self.generator.manual_seed(self.config["generator_seed"])
        else:
            self.generator.seed()

        self.model_dtype = model_dtype or torch.float32
        self.model_wrapper = self.model = model.to(dtype=self.model_dtype)
        self.model.enable_gradient_checkpointing()
        self.model.to(self.device)

        # until real encoders are loaded below, a truthy marker keeps get_conditions on the
        # "text provided" path for pre-encoded batches
        self.text_encoders = self.tokenizers = "pre-encoded"
        self._text_pending = pretrained_model_name_or_path
        self.vae = common_config.get("vae_instance")
        self.is_temporal_vae = bool(common_config.get("vae_is_temporal", False))
        # reference :953-958: class named by common_config["vae"] (default
        # "diffusers.AutoencoderKL"), loaded from <path>/vae; both map to the mirrors here
        vae_name = common_config.get("vae", "diffusers.AutoencoderKL")
        vae_path = common_config.get(
            "vae_pretrained_model_name_or_path", pretrained_model_name_or_path)
        if self.vae is None and vae_path is not None and \
                os.path.exists(os.path.join(vae_path, "vae", "config.json")):
            if vae_name.endswith("AutoencoderKLCogVideoX"):
                from dwm.models.cogvideox_vae import AutoencoderKLCogVideoX as vae_type
            elif vae_name.endswith("AutoencoderKL"):
                from dwm.models.autoencoder_kl import AutoencoderKL as vae_type
            else:
                raise Exception("Unsupported VAE type {}.".format(vae_name))
            self.vae = load_vae(vae_type, vae_path, common_config).to(self.device)
        if self.vae is not None and \
                type(self.vae).__name__ == "AutoencoderKLCogVideoX":
            self.is_temporal_vae = True

        self.is_dit = isinstance(self.model, _compat.SD3Transformer2DModelMarker)
        if self._text_pending is not None:       # real encoders when the checkpoint has them
            from dwm.pipelines.text_conditions import load_text_encoders
            loaded = load_text_encoders(
                self.is_dit, self._text_pending, self.device,
                common_config.get("text_encoder_load_args", {}),
                native=common_config.get("native_text_encoders", False))
            if loaded is not None:
                self.text_encoders, self.tokenizers = loaded
        if not self.is_dit and not isinstance(
                self.model, _compat.UNetSpatioTemporalConditionModelMarker):
            raise Exception("Unsupported diffusion model type.")
        default_scheduler = \
            "dwm.schedulers.temporal_independent.FlowMatchEulerDiscreteScheduler" \
            if self.is_dit else "dwm.schedulers.temporal_independent.DDIMScheduler"
        name = self.inference_config.get("scheduler", default_scheduler)
        # the reference's defaults / examples name diffusers classes; map them to mirrors
        name = {"diffusers.DDIMScheduler":
                "dwm.schedulers.temporal_independent.DDIMScheduler",
                "diffusers.DPMSolverMultistepScheduler":
                "dwm.schedulers.dpm_solver.DPMSolverMultistepScheduler",
                "diffusers.FlowMatchEulerDiscreteScheduler": default_scheduler}.get(
                    name, name)
        test_scheduler_type = dwm.common.get_class(name)
        sched_dir = None if pretrained_model_name_or_path is None else \
            os.path.join(pretrained_model_name_or_path, "scheduler")
        if sched_dir is not None and os.path.exists(
                os.path.join(sched_dir, "scheduler_config.json")):
            self.test_scheduler = test_scheduler_type.from_pretrained(
                pretrained_model_name_or_path, subfolder="scheduler")
        elif self.is_dit:
            # stable-diffusion-3.5-medium scheduler/scheduler_config.json values
            self.test_scheduler = test_scheduler_type(
                num_train_timesteps=1000, shift=3.0)
        else:
            # stable-diffusion-2-1 scheduler/scheduler_config.json values
            self.test_scheduler = test_scheduler_type(
                num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
                beta_schedule="scaled_linear", clip_sample=False,
                set_alpha_to_one=False, steps_offset=1,
                prediction_type="v_prediction")

        if resume_from is not None:
            self.model.load_state_dict(CrossviewTemporalSD.load_state(
                os.path.join(output_path, "checkpoints",
                             "{}.pth".format(resume_from))))
        elif model_checkpoint_path is not None:
            state_dict = CrossviewTemporalSD.load_state(model_checkpoint_path)
            missing_keys, unexpected_keys = self.model.load_state_dict(
                state_dict, **model_load_state_args)
            if self.should_save and \
                    self.common_config.get("print_load_state_info", False):
                print(f"missing keys: {missing_keys}")
                print(f"unexpected keys: {unexpected_keys}")
        self.metrics = metrics
        self._step_cache = {}
        # optional opendwm_b200.sharding.ShardPlan: this rank then owns one CFG branch /
        # a slice of the frames and `denoise_step` works on the local latents
        self.sharding = None

    @property
    def sharding(self):
        return getattr(self, "_sharding", None)

    @sharding.setter
    def sharding(self, plan):
        """Every rank of a sharded window must draw the same noise.  With `generator_seed`
        configured that holds by construction; otherwise rank 0's seed is broadcast when the
        plan is attached (the reference is single-process and has no such concern)."""
        self._sharding = plan
        if plan is not None and plan.world > 1 and \
                "generator_seed" not in (getattr(self, "config", None) or {}):
            import torch.distributed as dist
            if not dist.is_initialized():
                raise RuntimeError("a ShardPlan with world > 1 needs torch.distributed, or "
                                   "`generator_seed` in the pipeline config")
            box = [self.generator.initial_seed()]
            dist.broadcast_object_list(box, src=0)
            self.generator.manual_seed(box[0])

    # -- the fused denoising step ----------------------------------------------------------
    def _df_step_tensors(self, i, T, spi, take_time, B, V, frames=None):
        """Device-resident index tensors of one diffusion-forcing step, cached per
        (i, take_time): the reference rebuilds them from Python lists every step
        (:2048-2055, :2083-2088).  `frames` (a `ShardPlan.frame_slice()`) caches this
        rank's frames of them instead."""
        key = (i, T, spi, take_time, B, V, self.test_scheduler.num_inference_steps,
               None if frames is None else (frames.start, frames.stop))
        hit = self._step_cache.get(key)
        if hit is None and frames is not None:
            idx, timesteps, in_range = self._df_step_tensors(i, T, spi, take_time, B, V)
            hit = (idx[:, frames].contiguous(), timesteps[:, frames].contiguous(),
                   in_range[frames].contiguous())
            self._step_cache[key] = hit
        if hit is None:
            idx = torch.tensor(
                _ti.df_timestep_indices(i, T, spi, take_time),
                dtype=torch.int32, device=self.device)\
                .view(1, T, 1).repeat(B, 1, V).contiguous()
            timesteps = self.test_scheduler.timesteps.to(self.device)[idx.long()]
            in_range = torch.tensor(
                _ti.df_in_schedule_range(i, T, spi), device=self.device)\
                .to(torch.uint8).contiguous()
            hit = (idx, timesteps.float().contiguous(), in_range)
            self._step_cache[key] = hit
        return hit

    @torch.no_grad()
    def denoise_step(self, latents, conditions, idx, timesteps, in_range=None):
        """One iteration of the denoise loop (reference :2046-2090 /
        :1496-1575): CFG batching, noise-predict forward, CFG combine, per-frame Euler
        update and masked latent update.  `latents` fp32 [B,T,V,C,H,W] is updated in
        place; idx int32 [B,T,V]; timesteps fp32 [B,T,V]."""
        do_cfg = "guidance_scale" in self.inference_config
        if not self.is_dit:
            return self._denoise_step_unet(latents, conditions, timesteps, do_cfg)
        plan = self.sharding
        x = latents
        t = timesteps
        split_cfg = do_cfg and plan is not None and plan.cfg_ways == 2
        self.model.shard = plan
        tokens, _ = self.model.forward_tokens(
            x, t, conditions["encoder_hidden_states"],
            conditions["pooled_projections"],
            conditions.get("condition_image_tensor"),
            conditions.get("disable_crossview"),
            conditions.get("disable_temporal"),
            conditions.get("crossview_attention_mask"),
            conditions.get("added_time_ids"),
            t_offset=0 if plan is None else plan.t_offset,
            T_total=None if plan is None else plan.T,
            cfg_repeat=2 if (do_cfg and not split_cfg) else 1,
            v_offset=0 if plan is None else plan.v_offset,
            V_total=None if plan is None else plan.V)
        if split_cfg:   # exchange the branch predictions inside the CFG pair
            both = getattr(self, "_cfg_tokens", None)
            if both is None or both.shape[0] != 2 * tokens.shape[0]:
                both = self._cfg_tokens = torch.empty(
                    2 * tokens.shape[0], tokens.shape[1], device=tokens.device,
                    dtype=tokens.dtype)
            plan.gather_cfg_tokens(tokens, both)
            tokens = both
        sig = self.test_scheduler.sigmas
        if sig.device != latents.device:
            self.test_scheduler.sigmas = sig = sig.to(latents.device)
        _ops.cfg_euler_step(
            tokens, latents, idx, sig, cfg=2 if do_cfg else 1,
            guidance_scale=self.inference_config.get("guidance_scale", 1),
            patch=self.model.patch_size, in_range=in_range,
            round_dtype=self.model_dtype)
        return latents

    def denoise_step_graphed(self, latents, conditions, idx, timesteps, in_range=None):
        """`denoise_step` replayed from a CUDA graph (single GPU, fixed shapes and a fixed
        condition set): the small per-step tensors are copied into static buffers, the
        ~600 (UNet) / ~540 (DiT) launches of the step are submitted with one
        cudaGraphLaunch.  The first call per (latents, conditions) pair runs one eager
        warm-up step on a scratch copy (lazy weight packing, condition caches, workspace)
        and captures.

        A multistep scheduler (DPM-Solver++) is captured through its device-state protocol:
        the step's coefficient row is loaded into the scheduler's static row buffer before
        each replay and the host counters advance after it; the warm-up step and the capture
        leave the scheduler as they found it.  A multistep scheduler without that protocol
        runs eager."""
        sch = self.test_scheduler
        multistep = not self.is_dit and not hasattr(sch, "final_alpha_cumprod")
        device_state = multistep and hasattr(sch, "load_row")
        stateful = multistep and not device_state
        # sharded steps contain NCCL / symmetric-memory exchanges: captured only on request
        # (DWM_CUDA_GRAPH_SHARDED=1, not yet measured; DiT only, a sharded UNet step always
        # runs eager)
        sharded = self.sharding is not None and (
            not self.is_dit or os.environ.get("DWM_CUDA_GRAPH_SHARDED", "0") != "1")
        if self.sharding is not None and self.sharding.t_ways > 1 and \
                len(getattr(self.model, "temporal_block_layers", ())) % 2 == 1:
            # the peer K,V buffers alternate per temporal block; a captured step with an odd
            # number of blocks would end and restart on the same buffer (no barrier in between)
            sharded = True
        if self.sharding is not None and self.sharding.v_ways > 1 and \
                len(getattr(self.model, "crossview_block_layers", None) or ()) % 2 == 1:
            sharded = True          # the same for the view group's cross-view buffers
        if sharded or stateful:
            return self.denoise_step(latents, conditions, idx, timesteps, in_range)
        # the scheduler's history and row buffers are baked into the graph like the latents
        sch_bufs = sch.device_state(latents) if device_state else ()
        key = (latents.data_ptr(), tuple(latents.shape), idx is None, in_range is None,
               tuple(sorted((k, v.data_ptr(), tuple(v.shape), v._version)
                            for k, v in conditions.items() if torch.is_tensor(v))),
               tuple(b.data_ptr() for b in sch_bufs))
        graphs = self.__dict__.setdefault("_graphs", {})
        g = graphs.get(key)
        if g is None:
            st = dict(idx=None if idx is None else idx.clone(), ts=timesteps.clone(),
                      rng=None if in_range is None else in_range.clone())
            backup = latents.clone()
            sch_state = sch.snapshot() if device_state else None
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                self.denoise_step(latents, conditions, st["idx"], st["ts"], st["rng"])
            torch.cuda.current_stream().wait_stream(side)
            latents.copy_(backup)
            if device_state:
                sch.restore(sch_state)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                self.denoise_step(latents, conditions, st["idx"], st["ts"], st["rng"])
            if device_state:
                sch.restore(sch_state)
            # the entry keeps the keyed tensors alive (addresses are part of the key); a new
            # window / condition set means a new capture, so only the two most recent graphs
            # (and their private memory pools) are kept
            while len(graphs) >= 2:
                graphs.pop(next(iter(graphs)))
            g = graphs[key] = (graph, st, (latents, dict(conditions), sch_bufs))
        graph, st = g[:2]
        if idx is not None:
            st["idx"].copy_(idx)
        st["ts"].copy_(timesteps)
        if in_range is not None:
            st["rng"].copy_(in_range)
        if device_state:
            sch.load_row()
        graph.replay()
        if device_state:
            sch.advance()
        return latents

    def _denoise_step_unet(self, latents, conditions, timesteps, do_cfg):
        """CTSD-2.1 step: CFG batching, UNet forward, fused CFG + DDIM (eta 0) update
        (reference ctsd.py:1536-1575 with the in-repo DDIMScheduler.step).  Under a ShardPlan
        `latents` / `conditions` hold this rank's frames (and CFG branch, which the pair then
        exchanges); the update runs on the local frames."""
        plan = self.sharding
        split_cfg = do_cfg and plan is not None and plan.cfg_ways == 2
        self.model.shard = plan
        both = do_cfg and not split_cfg
        x = torch.cat([latents, latents]) if both else latents
        t = torch.cat([timesteps, timesteps]) if both else timesteps
        out, _, _ = self.model(
            x.to(self.model_dtype), t,
            encoder_hidden_states=conditions["encoder_hidden_states"],
            condition_image_tensor=conditions.get("condition_image_tensor"),
            disable_crossview=conditions.get("disable_crossview"),
            disable_temporal=conditions.get("disable_temporal"),
            crossview_attention_mask=conditions.get("crossview_attention_mask"),
            added_time_ids=conditions.get("added_time_ids"))
        pred = out[0].float().contiguous()
        if split_cfg:   # [uncond ; cond] predictions of the local frames on both ranks
            branch = pred
            pred = torch.empty((2 * branch.shape[0],) + tuple(branch.shape[1:]),
                               device=branch.device, dtype=branch.dtype)
            plan.gather_cfg_tokens(branch, pred)
        sch = self.test_scheduler
        if hasattr(sch, "cfg_step_"):
            # DPM-Solver++ multistep (reference :1573-1575, the scheduler counts steps itself):
            # CFG combine and update in one launch on the latents
            sch.cfg_step_(pred, latents, self.inference_config.get("guidance_scale", 1),
                          cfg=2 if do_cfg else 1)
            return latents
        if not hasattr(sch, "final_alpha_cumprod"):
            # any other scheduler: CFG combine, then its own scalar-timestep step
            if do_cfg:
                g = float(self.inference_config.get("guidance_scale", 1))
                w = self.__dict__.get("_cfg_w")
                if w is None or w[2] != g or w[0].device != pred.device:
                    w = self._cfg_w = (torch.tensor([1.0 - g], device=pred.device),
                                       torch.tensor([g], device=pred.device), g)
                u, c = pred[:pred.shape[0] // 2], pred[pred.shape[0] // 2:]
                pred = _ops.lincomb2(u.contiguous(), c.contiguous(), w[0], w[1],
                                     torch.empty_like(u))          # u + g (c - u)
            latents.copy_(sch.step(pred, timesteps.flatten()[0], latents).prev_sample)
            return latents
        sch.alphas_cumprod = sch.alphas_cumprod.to(latents.device)
        _ops.cfg_ddim_step(
            pred, latents,
            timesteps.to(torch.int32).contiguous(), sch.alphas_cumprod,
            cfg=2 if do_cfg else 1,
            guidance_scale=self.inference_config.get("guidance_scale", 1),
            step_ratio=sch.config.num_train_timesteps // sch.num_inference_steps,
            final_alpha_cumprod=float(sch.final_alpha_cumprod),
            prediction_type=sch.config.prediction_type, round_dtype=torch.float32)
        return latents

    def decode_latents(self, latents):
        """latents [n, C, h, w] -> images via the supplied VAE (reference :2092-2101);
        identity when no VAE object was configured."""
        if self.vae is None:
            return latents
        shift = self.vae.config.shift_factor \
            if self.vae.config.shift_factor is not None else 0
        return self.vae.decode(
            latents.to(dtype=self.vae.dtype) / self.vae.config.scaling_factor +
            shift, return_dict=False)[0]

    @staticmethod
    def postprocess(image_tensor, output_type="pt"):
        """diffusers VaeImageProcessor.postprocess for output_type "pt"/"latent":
        (x / 2 + 0.5).clamp(0, 1)."""
        if output_type not in ("pt", "latent"):
            raise NotImplementedError(
                "output_type {} needs PIL/numpy post-processing (outside the hot "
                "path); use \"pt\"".format(output_type))
        if output_type == "latent":
            return image_tensor
        return (image_tensor / 2 + 0.5).clamp(0, 1)

    @torch.no_grad()
    def inference_pipeline(self, latent_shape, batch, output_type,
                           image_latents=None, reference_frame_count: int = 0,
                           start_timestep: int = 0, stop_timestep=None,
                           take_time: int = 0):
        """Full-sequence (or diffusion-forcing) denoising of one window followed by the
        VAE decode — reference src/dwm/pipelines/ctsd.py:1439-1654 (the depth preview
        branch is dropped with the depth net, SURVEY.md §2 #14)."""
        df_mode = self.common_config.get("frame_prediction_style") == \
            "diffusion_forcing"
        steps = self.inference_config["inference_steps"]
        B, T, V = latent_shape[:3]
        if df_mode:
            clear = self.inference_config.get("clear_reference_frame_count", 0)
            assert steps % (T - clear) == 0
            spi = steps // (T - clear)
        self.test_scheduler.set_timesteps(steps, self.device)
        self._step_cache = {}
        if df_mode and image_latents is not None:
            latents = image_latents.to(self.device, torch.float32).clone()
        else:
            latents = torch.randn(tuple(latent_shape), generator=self.generator)\
                .to(self.device) * getattr(self.test_scheduler, "init_noise_sigma", 1)
        latents = latents.float().contiguous()
        conditions = CrossviewTemporalSD.get_conditions(
            self.model, self.text_encoders, self.tokenizers, self.common_config,
            latent_shape, batch, self.device, self.model_dtype,
            do_classifier_free_guidance="guidance_scale" in self.inference_config,
            latents_shape=latents.shape)
        stop_timestep = steps if stop_timestep is None else stop_timestep
        ts_table = self.test_scheduler.timesteps.to(self.device).float()
        inject = (not df_mode) and image_latents is not None and \
            reference_frame_count > 0
        # end-to-end sharding (opendwm_b200.sharding.ShardPlan in self.sharding): every rank
        # builds the full noise / conditions (same generator seed), keeps its CFG branch,
        # frames and views for the steps, and the window is re-assembled before the decode
        plan = self.sharding
        fs, vs = slice(0, T), slice(None)
        if plan is not None:
            fs, vs = plan.frame_slice(), plan.view_slice()
            conditions = plan.local_conditions(
                conditions, cfg_doubled="guidance_scale" in self.inference_config)
            latents = plan.local_latents(latents)
        # opt-in CUDA-graph replay of the step (inference_config["cuda_graph"] or env
        # DWM_CUDA_GRAPH=1): conditions are fixed for the whole window here
        use_graph = self.inference_config.get(
            "cuda_graph", os.environ.get("DWM_CUDA_GRAPH", "0") == "1")
        step = self.denoise_step_graphed if use_graph else self.denoise_step
        if hasattr(self.test_scheduler, "set_begin_index"):
            self.test_scheduler.set_begin_index(start_timestep)
        for i in range(start_timestep, stop_timestep):
            if df_mode:
                idx, timesteps, in_range = self._df_step_tensors(
                    i, T, spi, take_time, B, V)
            else:
                idx = torch.full((B, T, V), i, dtype=torch.int32, device=self.device)
                timesteps = ts_table[i].expand(B, T, V).contiguous()
                if not self.is_dit:
                    timesteps = timesteps.round().to(torch.int32)
                in_range = None
            if inject:
                # reference frames enter clean at timestep 0 and are restored after
                # the update, which reproduces the reference's per-step re-injection
                timesteps = timesteps.clone()
                timesteps[:, :reference_frame_count] = 0
                n_loc = max(0, min(reference_frame_count, fs.stop) - fs.start)
                if n_loc > 0:
                    latents[:, :n_loc] = \
                        image_latents[:, fs.start:fs.start + n_loc, vs].to(latents)
            if plan is not None:
                idx, timesteps = idx[:, fs, vs].contiguous(), timesteps[:, fs, vs].contiguous()
                in_range = None if in_range is None else in_range[fs].contiguous()
            step(latents, conditions, idx, timesteps, in_range)
        if plan is not None:
            latents = plan.gather_latents(latents)
        decode = self.decode_latents if plan is None or self.vae is None else \
            (lambda t: plan.split_call(self.decode_latents, t))
        if df_mode:
            cur = latents[:, take_time].flatten(0, 1)
            if self.is_temporal_vae and self.vae is not None:
                cur = torch.cat([cur[:, :, None], cur[:, :, None] * 0], dim=2)
                image_tensor = decode(cur).chunk(2, dim=2)[0]
                # "(b v) c t h w -> (b t v) c h w" (reference :1619-1621)
                image_tensor = image_tensor.unflatten(0, (B, V))\
                    .permute(0, 3, 1, 2, 4, 5).flatten(0, 2)
            else:
                image_tensor = decode(cur)
        else:
            if image_latents is not None:
                latents = torch.cat([
                    image_latents[:, :reference_frame_count].to(latents),
                    latents[:, reference_frame_count:]], 1)
            split = self.common_config.get("memory_efficient_batch", -1)
            if self.is_temporal_vae and self.vae is not None:
                # "b t v c h w -> (b v) c t h w"
                cur = latents.permute(0, 2, 3, 1, 4, 5).flatten(0, 1)
                image_tensor = dwm.functional.memory_efficient_split_call(
                    self, cur, lambda blk, t: blk.decode_latents(t), split) \
                    if plan is None else decode(cur)
                # "(b v) c t h w -> (b t v) c h w"
                Tn = image_tensor.shape[2]
                image_tensor = image_tensor.view(B, V, -1, Tn, *image_tensor.shape[-2:])\
                    .permute(0, 3, 1, 2, 4, 5).flatten(0, 2)
            else:
                image_tensor = dwm.functional.memory_efficient_split_call(
                    self, latents.flatten(0, 2),
                    lambda blk, t: blk.decode_latents(t), split) \
                    if plan is None else decode(latents.flatten(0, 2))
        images = image_tensor if self.vae is None else \
            CrossviewTemporalSD.postprocess(image_tensor, output_type)
        return {"images": images, "latents": latents}


    # -- long sequences: window after window ------------------------------------------------
    def get_latent_sequence_length(self, sequence_length):
        """Frames -> latent frames under a temporal VAE (`vae_pre` leading frames kept 1:1,
        the rest compressed by `vae_stride`); identity for image VAEs (reference :1113-1118)."""
        pre = self.inference_config.get("vae_pre", 0)
        stride = self.inference_config.get("vae_stride", 1)
        assert sequence_length % stride == pre or sequence_length == 0, \
            "{} vs {} vs {}".format(sequence_length, pre, stride)
        return (sequence_length - pre) // stride + (1 if pre > 0 else 0)

    def _window(self, batch, start, stop):
        keep = self.inference_config.get(
            "autoregression_data_exception_for_take_sequence", [])
        return {k: v if k in keep else dwm.functional.take_sequence_clip(v, start, stop)
                for k, v in batch.items()}

    @torch.no_grad()
    def autoregressive_inference_pipeline(self, latent_shape, batch, output_type):
        """Generates `batch["pts"].shape[1]` frames with windows of
        `sequence_length_per_iteration` frames (reference :1656-1833).

        Full-sequence style: every window re-uses the last `reference_frame_count` frames of
        the previous one as clean reference latents and contributes the frames after them.
        Diffusion-forcing style: the window is a queue of latents at staggered noise levels;
        a warm-up pass fills it, then every iteration runs `steps_per_inference` steps, emits
        the head frame, and (once `clear_reference_frame_count` heads are done) rotates the
        queue with a fresh noise frame at the tail; the tail is flushed at the end."""
        inf = self.inference_config
        n_total = batch["pts"].shape[1]
        win = inf["sequence_length_per_iteration"]
        n_ref = inf.get("reference_frame_count", 1)
        df_mode = self.common_config.get("frame_prediction_style") == "diffusion_forcing"
        image_latents = None
        if not inf.get("generate_frames_for_reference", True):
            # reference frames from real images: VAE-encode batch["vae_images"] (reference
            # :1677-1700).  Image VAEs only; the temporal-VAE encoder is not mirrored.
            if not hasattr(self.vae, "encode") or \
                    (self.is_temporal_vae and not hasattr(self.vae, "encoder")):
                raise NotImplementedError(
                    "reference frames from batch[\"vae_images\"] need a VAE encoder: "
                    "AutoencoderKL has one, AutoencoderKLCogVideoX only when built with "
                    "with_encoder=True (SURVEY.md §8(f)3)")
            raw = batch["vae_images"][:, :n_ref]
            x = raw.flatten(0, 2).to(self.device) * 2 - 1        # VaeImageProcessor.preprocess
            Bi, Ti, Vi = raw.shape[:3]
            if self.is_temporal_vae:      # "(b t v) c h w -> (b v) c t h w"
                x = x.unflatten(0, (Bi, Ti, Vi)).permute(0, 2, 3, 1, 4, 5).flatten(0, 1)
            shift = self.vae.config.shift_factor \
                if self.vae.config.shift_factor is not None else 0
            enc = dwm.functional.memory_efficient_split_call(
                self.vae, x.to(dtype=self.vae.dtype),
                lambda block, t: (block.encode(t).latent_dist.mode() - shift) *
                block.config.scaling_factor,
                self.common_config.get("memory_efficient_batch", -1))
            if self.is_temporal_vae:      # "(b v) c t h w -> b t v c h w"
                image_latents = enc.unflatten(0, (Bi, Vi)).permute(0, 3, 1, 2, 4, 5)
            else:
                image_latents = enc.unflatten(0, raw.shape[:3])
        images = []
        stride = win - n_ref
        starts = range(0, n_total - win + 1, stride)

        def has_next(i):
            return i + stride < n_total - win + 1

        if not df_mode:
            for i in starts:
                ref_now = 0 if image_latents is None else n_ref
                out = self.inference_pipeline(
                    latent_shape, self._window(batch, i, i + win), output_type, image_latents,
                    reference_frame_count=self.get_latent_sequence_length(ref_now))
                images.append(out["images"][latent_shape[0] * ref_now * latent_shape[2]:])
                if has_next(i):
                    image_latents = out["latents"][:, -self.get_latent_sequence_length(n_ref):]
        else:
            assert n_total > win
            steps = inf["inference_steps"]
            clear = inf.get("clear_reference_frame_count", 0)
            spi = steps // (latent_shape[1] - clear)
            T = latent_shape[1]

            def finished(head):      # queue slots whose frames are already final
                return torch.tensor([j <= head for j in range(T)], device=self.device)\
                    .view(1, T, 1, 1, 1, 1)
            # warm-up: bring the queue to the staggered steady state
            window = self._window(batch, 0, win)
            image_latents = self.inference_pipeline(
                latent_shape, window, output_type, image_latents, reference_frame_count=0,
                start_timestep=0, stop_timestep=steps - spi)["latents"]
            head = -1
            for i in starts:
                window = self._window(batch, i, i + win)
                ref_now = n_ref
                if head < clear:
                    ref_now = T
                    head += 1
                out = self.inference_pipeline(
                    latent_shape, window, output_type, image_latents,
                    reference_frame_count=ref_now,
                    start_timestep=steps + (head - 1) * spi,
                    stop_timestep=steps + head * spi, take_time=head)
                images.append(out["images"].chunk(4)[-1]
                              if self.is_temporal_vae and i == 0 else out["images"])
                image_latents = torch.where(finished(head), image_latents, out["latents"])
                if head == clear and has_next(i):
                    fresh = torch.randn((latent_shape[0], 1) + tuple(latent_shape[2:]),
                                        generator=self.generator).to(self.device) * \
                        getattr(self.test_scheduler, "init_noise_sigma", 1)
                    image_latents = torch.cat([image_latents[:, 1:], fresh], 1)
            for j in range(head + 1, T):       # flush: the last window keeps its conditions
                out = self.inference_pipeline(
                    latent_shape, window, output_type, image_latents, reference_frame_count=T,
                    start_timestep=steps + (j - 1) * spi, stop_timestep=steps + j * spi,
                    take_time=j)
                images.append(out["images"])
                image_latents = torch.where(finished(j), image_latents, out["latents"])
        return {"images": torch.cat(images) if output_type == "pt" else images}


    # -- entry point of src/dwm/preview.py ------------------------------------------------------
    def _preview_latent_shape(self, batch, frames):
        """[B, latent frames, V, C, h, w] from the batch's image size and the VAE config
        (reference :1839-1862, :2283-2294)."""
        B, _, V = batch["vae_images"].shape[:3]
        down = 2 ** (len(self.vae.config.down_block_types) - 1)
        return (B, frames, V, self.vae.config.latent_channels,
                batch["vae_images"].shape[-2] // down, batch["vae_images"].shape[-1] // down)

    def _dump_preview(self, images, batch, output_path, global_step):
        """Writes <output_path>/preview/<step>.png|.mp4 through the reference's
        dwm.utils.preview (PyAV based, not part of this mirror) when it is importable — i.e.
        when these files are overlaid on the reference tree — and PNG frames otherwise."""
        import torchvision
        all_rank = self.inference_config.get("all_rank_preview", False)
        if not (self.should_save or (torch.distributed.is_initialized() and all_rank)):
            return
        folder = os.path.join(output_path, "preview")
        os.makedirs(folder, exist_ok=True)
        name = "{}_{}".format(global_step, torch.distributed.get_rank()) if all_rank \
            else str(global_step)
        frames = batch["vae_images"].shape[1]
        try:
            import dwm.utils.preview as up
            tensor = up.make_ctsd_preview_tensor(images, batch, self.inference_config)
            if frames == 1:
                torchvision.transforms.functional.to_pil_image(tensor).save(
                    os.path.join(folder, name + ".png"))
            else:
                up.save_tensor_to_video(os.path.join(folder, name + ".mp4"), "libx264",
                                        batch["fps"][0].item(), tensor)
        except ImportError:
            B, _, V = batch["vae_images"].shape[:3]
            grid = images.float().cpu().unflatten(0, (B, -1, V))
            for t in range(grid.shape[1]):
                torchvision.utils.save_image(
                    grid[:, t].flatten(0, 1), os.path.join(
                        folder, name + (".png" if grid.shape[1] == 1 else "_%04d.png" % t)),
                    nrow=V)

    @torch.no_grad()
    def preview_pipeline(self, batch: dict, output_path: str, global_step: int):
        """Generates the whole clip of `batch` (autoregressively when
        `sequence_length_per_iteration` is configured) and dumps it (reference :1836-1897)."""
        n = batch["vae_images"].shape[1]
        if "sequence_length_per_iteration" in self.inference_config:
            shape = self._preview_latent_shape(batch, self.get_latent_sequence_length(
                self.inference_config["sequence_length_per_iteration"]))
            out = self.autoregressive_inference_pipeline(shape, batch, "pt")
        else:
            shape = self._preview_latent_shape(batch, self.get_latent_sequence_length(n))
            out = self.inference_pipeline(shape, batch, "pt")
        self._dump_preview(out["images"], batch, output_path, global_step)
        return out


class StreamingCrossviewTemporalSD(CrossviewTemporalSD):

    def reset_streaming(self, latent_shape, output_type):
        assert self.common_config.get("frame_prediction_style") == \
            "diffusion_forcing"
        self.conditions = {}
        self.condition_count = 0
        self.latents = None
        self.text_prompt_counter = 0
        self.frames = []
        self.latent_shape = tuple(latent_shape)
        self.output_type = output_type
        self.test_scheduler.set_timesteps(
            self.inference_config["inference_steps"], self.device)
        self.prev_ego_transforms = None
        self._step_cache = {}
        self._local_conditions = None
        self._streaming_plan()

    def _streaming_plan(self):
        """The ShardPlan of the streaming steps, or None.  Sharding is DiT-only: a UNet
        pipeline with a plan is refused rather than run unsharded on every rank."""
        plan = self.sharding
        if plan is not None and not self.is_dit:
            raise NotImplementedError(
                "StreamingCrossviewTemporalSD.sharding needs the DiT model: the CTSD-2.1 UNet "
                "step is not sharded; detach the ShardPlan (pipe.sharding = None)")
        return plan

    @torch.no_grad()
    def inference_pipeline(self, latent_shape, start_timestep: int = 0,
                           stop_timestep=None, take_time: int = 0):
        """reference :2031-2103.

        With a ShardPlan every rank holds the whole FIFO (`self.latents`, `self.conditions`);
        a call runs its steps on this rank's CFG branch and frames and all-gathers the FIFO
        once at the end.  The exiting frame's views are decoded item-parallel over all
        ranks, so every rank emits the same frame."""
        steps = self.inference_config["inference_steps"]
        assert steps % latent_shape[1] == 0
        spi = steps // latent_shape[1]
        B, T, V = latent_shape[:3]
        latents = self.latents.to(torch.float32).contiguous()
        stop_timestep = stop_timestep or steps
        plan = self._streaming_plan()
        conditions, fs, decode, work = self.conditions, None, self.decode_latents, latents
        V_work = V
        if plan is not None:
            if plan.T != T:
                raise ValueError("the ShardPlan splits {} frames, the FIFO holds {}".format(
                    plan.T, T))
            if plan.V is not None and plan.V != V:
                raise ValueError("the ShardPlan splits {} views, the FIFO holds {}".format(
                    plan.V, V))
            # sliced once per condition update: the flush reuses one condition set, and the
            # model's condition cache is keyed by tensor address
            if self._local_conditions is None or self._local_conditions[0] is not plan:
                self._local_conditions = (plan, plan.local_conditions(
                    self.conditions, cfg_doubled="guidance_scale" in self.inference_config))
            conditions, fs = self._local_conditions[1], plan.frame_slice()
            work = plan.local_latents(latents)
            V_work = work.shape[2]
            if self.vae is not None:
                decode = lambda t: plan.split_call(self.decode_latents, t)  # noqa: E731
        for i in range(start_timestep, stop_timestep):
            idx, timesteps, in_range = self._df_step_tensors(
                i, T, spi, take_time, B, V_work, frames=fs)
            self.denoise_step(work, conditions, idx, timesteps, in_range)
        if plan is not None:
            # unsharded, the steps update `latents` in place, and an fp32 FIFO is `latents`
            # itself (so in the flush its finished slots keep the extra steps): the gathered
            # FIFO goes to the same tensor, and both paths leave the same `self.latents`
            latents.copy_(plan.gather_latents(work))
        if stop_timestep >= steps:
            # reference :2092-2101: VAE decode of the exiting frame, then
            # image_processor.postprocess(image_tensor, self.output_type)
            image_tensor = decode(latents[:, take_time].flatten(0, 1))
            self.frames.append(
                image_tensor if self.vae is None else
                CrossviewTemporalSD.postprocess(image_tensor, self.output_type))
        return latents

    @torch.no_grad()
    def send_frame_condition(self, frame_condition_data):
        """reference :2105-2219."""
        do_cfg = "guidance_scale" in self.inference_config
        steps = self.inference_config["inference_steps"]
        spi = steps // self.latent_shape[1]
        seq = self.inference_config["sequence_length_per_iteration"]
        if frame_condition_data is None:      # flushing
            assert self.condition_count == seq
            for i in range(1, self.latent_shape[1]):
                latents = self.inference_pipeline(
                    self.latent_shape, start_timestep=steps + (i - 1) * spi,
                    stop_timestep=steps + i * spi, take_time=i)
                is_finished = torch.tensor(
                    [j <= i for j in range(self.latent_shape[1])],
                    device=self.device).view(1, -1, 1, 1, 1, 1)
                self.latents = torch.where(is_finished, self.latents, latents)
            return

        fc = CrossviewTemporalSD.get_conditions(
            self.model,
            self.text_encoders if self.text_prompt_counter == 0 else None,
            self.tokenizers, self.common_config,
            (self.latent_shape[0], 1) + tuple(self.latent_shape[2:]),
            frame_condition_data, self.device, self.model_dtype,
            streaming_mode=True, prev_ego_transforms=self.prev_ego_transforms,
            do_classifier_free_guidance=do_cfg)
        if "ego_transforms" in frame_condition_data:
            self.prev_ego_transforms = frame_condition_data["ego_transforms"]
        if self.text_prompt_counter > 0:
            fc["encoder_hidden_states"] = \
                self.conditions["encoder_hidden_states"][:, -1:]
            fc["pooled_projections"] = \
                self.conditions["pooled_projections"][:, -1:]
        self.text_prompt_counter = (self.text_prompt_counter + 1) % \
            self.inference_config.get("text_prompt_interval", 1)
        keep = self.inference_config[
            "autoregression_condition_exception_for_take_sequence"]
        noise_scale = getattr(self.test_scheduler, "init_noise_sigma", 1)
        self._local_conditions = None          # a ShardPlan re-slices the new condition set
        if self.condition_count < seq:        # gathering
            for k, v in fc.items():
                if k not in self.conditions or k in keep or v is None:
                    self.conditions[k] = v
                else:
                    self.conditions[k] = torch.cat([self.conditions[k], v], dim=1)
            self.condition_count += 1
            if self.condition_count == seq:
                self.latents = torch.randn(
                    self.latent_shape, generator=self.generator)\
                    .to(self.device) * noise_scale
                self.latents = self.inference_pipeline(
                    self.latent_shape, start_timestep=0, stop_timestep=steps)
        else:                                  # streaming
            for k, v in fc.items():
                if k not in self.conditions or k in keep or v is None:
                    self.conditions[k] = v
                else:
                    self.conditions[k] = torch.cat(
                        [self.conditions[k][:, 1:], v], dim=1)
            # tell the model that the new condition set is the previous one moved on by a
            # frame, so that it updates its step-invariant cache incrementally (equal to the
            # full rebuild: tests/test_model_gpu.py::test_streaming_ring_cache_equals_full_
            # recompute); `condition_ring: false` / DWM_STREAM_RING=0 switches it off
            if self.inference_config.get(
                    "condition_ring", os.environ.get("DWM_STREAM_RING", "1") == "1"):
                self.model._ring_shift = True
            self.latents = torch.cat([
                self.latents[:, 1:],
                torch.randn((self.latent_shape[0], 1) + self.latent_shape[2:],
                            generator=self.generator).to(self.device) *
                noise_scale], 1)
            self.latents = self.inference_pipeline(
                self.latent_shape, start_timestep=steps - spi,
                stop_timestep=steps)

    def receive_frame(self):
        if len(self.frames) == 0:
            return None
        return self.frames.pop(0)

    def fifo_inference_pipeline(self, latent_shape, batch, output_type):
        """reference :2234-2277."""
        total_frame_count = batch["pts"].shape[1]
        assert total_frame_count > \
            self.inference_config["sequence_length_per_iteration"]
        skip = self.inference_config[
            "autoregression_data_exception_for_take_sequence"]
        result = {"images": []}
        self.reset_streaming(latent_shape, output_type)
        for i in range(total_frame_count):
            self.send_frame_condition({
                k: (v if k in skip
                    else dwm.functional.take_sequence_clip(v, i, i + 1))
                for k, v in batch.items()})
            image = self.receive_frame()
            if image is not None:
                result["images"].append(image)
        self.send_frame_condition(None)
        while True:
            image = self.receive_frame()
            if image is None:
                break
            result["images"].append(image)
        if output_type == "pt":
            result["images"] = torch.cat(result["images"])
        return result

    @torch.no_grad()
    def preview_pipeline(self, batch: dict, output_path: str, global_step: int):
        """FIFO generation of the whole clip (reference :2280-2330)."""
        assert "sequence_length_per_iteration" in self.inference_config
        shape = self._preview_latent_shape(
            batch, self.inference_config["sequence_length_per_iteration"])
        out = self.fifo_inference_pipeline(shape, batch, "pt")
        self._dump_preview(out["images"], batch, output_path, global_step)
        return out
