"""``create_gaussian_diffusion`` and ``create_gaussian_diffusion_ddpm`` — the yaml ``diffusion.target`` factories, same
keyword-only signatures as the reference (reference models/script_util.py:7-92)."""
from __future__ import annotations

from . import gaussian_diffusion as gd


def create_gaussian_diffusion(*, normalize_input, schedule_name, sf=4, min_noise_level=0.01, steps=1000, kappa=1,
                              etas_end=0.99, schedule_kwargs=None, weighted_mse=False, predict_type="xstart",
                              timestep_respacing=None, scale_factor=None, latent_flag=True):
    sqrt_etas = gd.get_named_eta_schedule(schedule_name, num_diffusion_timesteps=steps,
                                          min_noise_level=min_noise_level, etas_end=etas_end, kappa=kappa,
                                          kwargs=schedule_kwargs)
    if timestep_respacing is None:
        timestep_respacing = steps
    else:
        assert isinstance(timestep_respacing, int)
    try:
        mean_type = {"xstart": gd.ModelMeanType.START_X, "epsilon": gd.ModelMeanType.EPSILON,
                     "epsilon_scale": gd.ModelMeanType.EPSILON_SCALE, "residual": gd.ModelMeanType.RESIDUAL}[predict_type]
    except KeyError:
        raise ValueError(f"Unknown Predicted type: {predict_type}")
    return gd.ResShiftDiffusion(
        use_timesteps=gd.space_timesteps(steps, timestep_respacing), sqrt_etas=sqrt_etas, kappa=kappa,
        model_mean_type=mean_type, loss_type=gd.LossType.WEIGHTED_MSE if weighted_mse else gd.LossType.MSE,
        scale_factor=scale_factor, normalize_input=normalize_input, sf=sf, latent_flag=latent_flag)


def create_gaussian_diffusion_ddpm(*, beta_start, beta_end, sf=4, steps=1000, learn_sigma=False, sigma_small=False,
                                   noise_schedule="linear", predict_xstart=False, timestep_respacing=None,
                                   scale_factor=1.0):
    """The DDPM / DDIM process (reference models/script_util.py:57-92)."""
    betas = gd.get_named_beta_schedule(noise_schedule, steps, beta_start, beta_end)
    if timestep_respacing is None:
        timestep_respacing = steps
    else:
        assert isinstance(timestep_respacing, int)
    if learn_sigma:
        var_type = gd.ModelVarTypeDDPM.LEARNED_RANGE
    else:
        var_type = gd.ModelVarTypeDDPM.FIXED_SMALL if sigma_small else gd.ModelVarTypeDDPM.FIXED_LARGE
    return gd.SpacedDiffusionDDPM(
        use_timesteps=gd.space_timesteps(steps, timestep_respacing), betas=betas,
        model_mean_type=gd.ModelMeanType.START_X if predict_xstart else gd.ModelMeanType.EPSILON,
        model_var_type=var_type, scale_factor=scale_factor, sf=sf)
