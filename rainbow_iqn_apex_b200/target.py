"""The EMA target network (BBF, Schwarzer et al., "Bigger, Better, Faster: Human-level Atari with human-level
efficiency", ICML 2023): under ``target_ema`` the learner moves the target network towards the online one after every
update, xi <- xi + tau (theta - xi), instead of leaving it to the caller's periodic hard copy.

After every optimiser's step and the side networks' after_step hooks, one riqn_ema_f32 launch runs over the whole
online parameter arena into the target's (each operation rounded on its own), and the target's cached operand images
(conv / iqn_fc) are marked stale, so that the next step's target pass rebuilds them from the new weights.  Every step
entry point reaches this through Learner._step_optimisers, and so does every captured step graph, whose capture forces
the rebuild as it does the online network's.

Left alone: the target's epsilon arena (the target draws its own noise every pass), update_target_net() (still a hard
copy, from which the EMA continues), resets (the target follows the reset online network at rate tau) and CURL's
momentum encoder (its own tau).  Data-parallel replicas hold the same online arena after the all-reduce and the step,
so each runs the same EMA without a collective; under Ape-X only the learner rank has a target.
"""
from ._lib import call, ptr


def update(learner):
    """xi <- xi + tau (theta - xi) over the whole online arena, when target_ema is on."""
    if learner.target_ema is None:
        return
    on, tg = learner.online_net, learner.target_net
    call("riqn_ema_f32", on._flat.numel(), ptr(on._flat), ptr(tg._flat), learner.target_ema)
    tg._params_changed()
