"""megaverse_b200: H100-native batched voxel-world step + render engine behind the Megaverse env API.

Only the per-step hot path is here (agent kinematics + collision, carry/place, reward/done, first-person rasteriser);
see DESIGN.md.  `MegaverseEnv` mirrors megaverse/megaverse_env.py of the reference."""

__all__ = ["MegaverseEnv", "make_env_multitask", "make_env_mixed", "MEGAVERSE8"]


def __getattr__(name):
    if name in __all__:
        from . import megaverse_env

        return getattr(megaverse_env, name)
    raise AttributeError(name)
