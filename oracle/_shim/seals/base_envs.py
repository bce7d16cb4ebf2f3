"""Names-only stub (oracle/_shim): `seals.base_envs.TabularModelPOMDP`, which the reference's algorithms/mce_irl.py names
in annotations only; MCE IRL reads the env's attributes (oracle/tabular_mdp.py supplies them)."""


class TabularModelPOMDP:
    pass
