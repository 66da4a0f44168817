"""Human3.6M action names for actionwise evaluation -- mirror of `define_actions` in the
reference lib/utils/data_utils.py (:325-347); the rest of that module is dataset preparation."""

ACTIONS = ["Directions", "Discussion", "Eating", "Greeting", "Phoning", "Photo", "Posing", "Purchases",
           "Sitting", "SittingDown", "Smoking", "Waiting", "WalkDog", "Walking", "WalkTogether"]


def define_actions(action):
    """'All' / 'all' -> the 15 actions; one action name -> [name]; anything else: ValueError."""
    if action in ("All", "all"):
        return list(ACTIONS)
    if action not in ACTIONS:
        raise ValueError("Unrecognized action: %s" % action)
    return [action]
