"""Event functions: markers only.  The fused-step env lowers them by name onto wl_startup / the fused step
(a13, a14 in SURVEY 8a); calling them directly is not supported."""


def _marker(name):
    def f(env, env_ids, *args, **kwargs):
        raise NotImplementedError(f"isaaclab.envs.mdp.{name} is executed inside the fused CUDA step; it is a marker here")
    f.__name__ = name
    f.__qualname__ = name
    return f


randomize_rigid_body_material = _marker("randomize_rigid_body_material")
randomize_actuator_gains = _marker("randomize_actuator_gains")
randomize_rigid_body_mass = _marker("randomize_rigid_body_mass")
push_by_setting_velocity = _marker("push_by_setting_velocity")
reset_root_state_uniform = _marker("reset_root_state_uniform")
reset_scene_to_default = _marker("reset_scene_to_default")
