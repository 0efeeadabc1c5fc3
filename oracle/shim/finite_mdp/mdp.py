"""`finite_mdp.mdp.DeterministicMDP` as a plain record of its constructor arguments (no solver)."""


class DeterministicMDP:
    mode = "deterministic"

    def __init__(self, transition, reward, terminal=None, state=0):
        self.transition = transition
        self.reward = reward
        self.terminal = terminal
        self.state = state
