from crowdnav_prediction_attngraph_b200.gym_env import CrowdSimPred, CrowdSimVarNum, CrowdSimPredRealGST, \
    CrowdSimVarNumCollect  # noqa: F401
