/*
 * hwyb200.h — C ABI of the H100-native batched HighwayEnv hot path.
 *
 * Plain pointers and sizes only (no torch / C++ types).  Every pointer in the *State
 * structs and every array argument is a DEVICE pointer owned by the caller (the Python
 * host allocates them as torch CUDA tensors); kernels run on the `stream` argument
 * (a cudaStream_t passed as void*, NULL = legacy default stream) and never allocate.
 * All functions return 0 on success, non-zero on error (hwy_last_error() gives the text);
 * there is no CPU fallback anywhere behind this interface.
 *
 * The reference (HighwayEnv 1.12.1, pure Python) has no FFI; the seam these entry points
 * replace is the operator interface AbstractEnv._simulate drives
 * (highway_env/envs/common/abstract.py:287-317):
 *     action_type.act(action); road.act(); road.step(1 / simulation_frequency)
 * followed by observation_type.observe(), _reward(), _is_terminated(), _is_truncated()
 * (abstract.py:277-280), and AbstractEnv.reset()'s _reset() (abstract.py:219-249).
 * INTEGRATION.md shows the ctypes binding a reference maintainer would add.
 */
#ifndef HWYB200_H
#define HWYB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HWY_ABI_VERSION 17
#define HWY_MAX_LANES 8
#define HWY_MAX_TARGET_SPEEDS 8
#define HWY_MAX_VEHICLES 128 /* per env, incl. the ego */
#define HWY_MAX_OBS_VEHICLES 16
#define HWY_REWARD_TERMS 5 /* slots of the reward_terms rows (info["rewards"]) */

/* vehicle kinds (bits 19-20 of `meta`) */
#define HWY_KIND_IDM 0     /* highway_env/vehicle/behavior.py:12   IDMVehicle */
#define HWY_KIND_MDP 1     /* highway_env/vehicle/controller.py:256 MDPVehicle */
#define HWY_KIND_VEHICLE 2 /* highway_env/vehicle/kinematics.py:13  Vehicle */

/* meta word layout (one int32 per vehicle slot) */
#define HWY_META_LANE_SHIFT 0         /* 8 bits: lane_index (graph enumeration order) */
#define HWY_META_TARGET_SHIFT 8       /* 8 bits: target_lane_index */
#define HWY_META_CRASHED (1 << 16)
#define HWY_META_HAS_IMPACT (1 << 17) /* Vehicle.impact is not None */
#define HWY_META_CHECK_COLLISIONS (1 << 18)
#define HWY_META_KIND_SHIFT 19        /* 2 bits */
#define HWY_META_PRESENT (1 << 21)
/* highway family only, 7 bits: the slot of the env's vehicle of rank v along the road (v = this slot's index) as of
 * the last frame a highway kernel built, or after a spawn whose positions increase with the slot.  A hint for the next
 * step's first frame, which checks it against the positions before using it: any value is safe, and the reset value
 * 0 in every slot (what a state written from the host has) just means "recount". */
#define HWY_META_ORDER_SHIFT 24
/* kinds (2 bits): 0 IDMVehicle, 1 MDPVehicle, 2 plain Vehicle (ContinuousAction ego), 3 Obstacle — a static 2 x 2 m
 * road object (vehicle/objects.py:213-220); road.objects occupy the slots after the vehicles */
#define HWY_KIND_OBSTACLE 3

/* Kinematics feature columns (Vehicle.to_dict keys, vehicle/kinematics.py:240-254) */
#define HWY_MAX_OBS_FEATURES 16
#define HWY_FEAT_PRESENCE 0
#define HWY_FEAT_X 1
#define HWY_FEAT_Y 2
#define HWY_FEAT_VX 3
#define HWY_FEAT_VY 4
#define HWY_FEAT_HEADING 5
#define HWY_FEAT_COS_H 6
#define HWY_FEAT_SIN_H 7
#define HWY_FEAT_COS_D 8
#define HWY_FEAT_SIN_D 9
#define HWY_FEAT_LONG_OFF 10
#define HWY_FEAT_LAT_OFF 11
#define HWY_FEAT_ANG_OFF 12

/* autoreset modes of hwy_highway_step (gymnasium.vector.AutoresetMode) */
#define HWY_AUTORESET_DISABLED 0
#define HWY_AUTORESET_SAME_STEP 1 /* reset inside the step that ended; obs = reset obs */

/* A StraightLane (highway_env/road/lane.py:159-213), fields as its __init__ computes them. */
typedef struct HwyStraightLane {
    double start_x, start_y;
    double dir_x, dir_y;         /* direction */
    double lat_x, lat_y;         /* direction_lateral */
    double heading, length, width, speed_limit;
} HwyStraightLane;

/* Scenario parameters of the straight multi-lane highway family: highway-v0 and
 * highway-fast-v0 (highway_env/envs/highway_env.py:25-53,162-182 over
 * envs/common/abstract.py:102-125).  Passed by value to the kernels. */
typedef struct HwyHighwayParams {
    int32_t lanes_count;
    int32_t n_vehicles;              /* controlled (1) + vehicles_count, <= HWY_MAX_VEHICLES */
    int32_t simulation_frequency;
    int32_t policy_frequency;
    int32_t action_type;             /* 0 DiscreteMetaAction (action.py:199-298), 1 ContinuousAction (:73-162) */
    int32_t others_check_collisions; /* 0 = highway-fast-v0 (highway_env.py:177-182) */
    int32_t normalize_reward;
    int32_t offroad_terminal;
    int32_t obs_vehicles_count;      /* KinematicObservation.vehicles_count (observation.py:163) */
    int32_t obs_see_behind;
    int32_t obs_absolute;
    int32_t obs_normalize;
    int32_t obs_clip;
    int32_t n_target_speeds;
    int32_t initial_lane_id;         /* -1 = None */
    int32_t act_clip;                /* ContinuousAction.clip */
    double duration;
    double target_speeds[HWY_MAX_TARGET_SPEEDS]; /* MDPVehicle.target_speeds (controller.py:259) */
    double collision_reward, right_lane_reward, high_speed_reward;
    double reward_speed_lo, reward_speed_hi;
    double acc_lo, acc_hi, steer_lo, steer_hi;   /* action.py:82-86 */
    double ego_spacing, vehicles_density, ego_speed;
    double spawn_exp;                /* np.exp(-5/40*lanes) evaluated on the host (kinematics.py:95) */
    /* IDM / MOBIL (behavior.py:21-46) */
    double acc_max, comfort_acc_max, comfort_acc_min, distance_wanted, time_wanted;
    double politeness, lane_change_min_acc_gain, lane_change_max_braking_imposed, lane_change_delay;
    double delta_lo, delta_hi;
    double perception_distance;      /* abstract.py:56 */
    HwyStraightLane lanes[HWY_MAX_LANES];
    /* KinematicObservation.features / features_range (observation.py:160-232; Vehicle.to_dict,
     * vehicle/kinematics.py:237-261).  obs_n_features == 0: the default columns (presence, x, y, vx, vy)
     * with the default ranges.  Otherwise column c holds feature obs_feature[c] (HWY_FEAT_*), mapped
     * from [obs_feature_lo, obs_feature_hi] to [-1, 1] when obs_normalize and obs_feature_ranged[c]. */
    int32_t obs_n_features;
    /* config["controlled_vehicles"] (0 or 1: one controlled vehicle; at most 8).  With n_agents > 1 the step, reset
     * and observe entry points run the multi-agent kernels: the controlled vehicles sit at the slots
     * _create_vehicles gives them (highway_env.py:72-98): bin k of near_split(n_vehicles - n_agents, n_agents)
     * (utils.py:355) is controlled vehicle k followed by its traffic.  Agent k of a step is the k-th slot whose kind
     * is HWY_KIND_MDP or HWY_KIND_VEHICLE; speed_index holds [n_envs][n_agents]; reward, flags and info are the
     * first controlled vehicle's (slot 0).  LinearVehicle traffic is refused with n_agents > 1.
     *   multi_action (MultiAgentAction, action.py:301-333): action_i [n_envs][n_agents] or action_f
     *     [n_envs][n_agents][2], one action per controlled vehicle.  0: action_i [n_envs] / action_f [n_envs][2] go
     *     to the first one and the others act(None): IDLE for an MDPVehicle, the kept {0, 0} for a plain Vehicle.
     *   multi_obs (MultiAgentObservation, observation.py:588-604): the Kinematics observation is written once per
     *     controlled vehicle as observer, obs [n_envs][n_agents][K][columns].  0: the first one's, [n_envs][K][..]. */
    int16_t n_agents;
    uint8_t multi_action, multi_obs;
    int32_t obs_feature[HWY_MAX_OBS_FEATURES];
    int32_t obs_feature_ranged[HWY_MAX_OBS_FEATURES];
    double obs_feature_lo[HWY_MAX_OBS_FEATURES], obs_feature_hi[HWY_MAX_OBS_FEATURES];
} HwyHighwayParams;

/* Device-resident state of n_envs independent roads, structure of arrays over
 * (env, vehicle slot); slot stride `vp` (see hwy_highway_slot_stride).  Packed pairs are
 * interleaved doubles so that one thread moves one vehicle with 128-bit accesses.
 *   pos[2*(e*vp+v)+{0,1}] = position x, y         hs = heading, speed
 *   tt  = target_speed, timer (IDM lane-change timer) imp = Vehicle.impact x, y
 * Per env: speed_index (MDPVehicle.speed_index), time (AbstractEnv.time), and the numpy
 * Generator(PCG64) stream of env.np_random as 5 words rng[k*n_envs+e]:
 *   k=0 state_hi, 1 state_lo, 2 inc_hi, 3 inc_lo, 4 (has_uint32 << 32) | uinteger. */
typedef struct HwyHighwayState {
    int32_t n_envs;
    int32_t vp;
    double *pos, *hs, *tt, *imp; /* [n_envs*vp*2] */
    double *delta;               /* [n_envs*vp]   IDMVehicle.DELTA */
    int32_t *meta;               /* [n_envs*vp] */
    int32_t *speed_index;        /* [n_envs * max(1, n_agents)] MDPVehicle.speed_index of each controlled vehicle */
    double *time;                /* [n_envs] */
    uint64_t *rng;               /* [5*n_envs] */
    double *reward_terms;        /* [n_envs*HWY_REWARD_TERMS] or NULL: the un-weighted terms of AbstractEnv._rewards
                                  * (info["rewards"], abstract.py:213-216) of the step, before any autoreset.
                                  * highway: collision, right_lane, high_speed, on_road (highway_env.py:118-137) */
} HwyHighwayState;

int hwy_abi_version(void);
const char *hwy_last_error(void);

/* Slot stride for n_vehicles (next multiple of 2; 128-bit alignment of the packed pairs). */
int hwy_highway_slot_stride(int n_vehicles);

/* LinearVehicle traffic (vehicle/behavior.py:350-583; AggressiveVehicle and DefensiveVehicle
 * are the same model on the highway, they differ only in p->lane_change_min_acc_gain).  Every
 * traffic vehicle keeps the parameters randomize_behavior drew for it (behavior.py:406-415):
 *   params[5*(e*vp+v) + 0..2] = ACCELERATION_PARAMETERS, + 3..4 = STEERING_PARAMETERS
 * (DEVICE, [n_envs*vp*5] doubles; the controlled vehicle's row is zero).  A reset draws
 *   ACCELERATION_PARAMETERS = acc_lo + uniform(size=3) * acc_span,
 *   STEERING_PARAMETERS     = steer_lo + uniform(size=2) * steer_span
 * with acc_lo = ACCELERATION_RANGE[0], acc_span = ACCELERATION_RANGE[1] - ACCELERATION_RANGE[0]
 * (likewise steering) as numpy evaluates them on the host.  p->time_wanted is the class's
 * TIME_WANTED (2.5).  The reset, step and substeps entry points below take a `t` argument:
 * NULL runs IDMVehicle traffic, non-NULL (with t->params set) runs this traffic model. */
#define HWY_LINEAR_PARAMS 5
typedef struct HwyLinearTraffic {
    double *params;
    double acc_lo[3], acc_span[3];
    double steer_lo[2], steer_span[2];
} HwyLinearTraffic;

/* AbstractEnv.reset()'s _reset() for the envs with mask_a[e] | mask_b[e] (both NULL: every
 * env): HighwayEnv._create_road/_create_vehicles (highway_env.py:55-98,177-182) with
 * Vehicle.create_random (kinematics.py:50-104), drawing from each env's PCG64 stream in
 * the reference's order.  If obs != NULL also writes the reset observation
 * [n_envs][obs_vehicles_count][n columns] float32 of those envs.  With mask_a = terminated
 * and mask_b = truncated this is the SameStep autoreset half of hwy_highway_step on its own
 * (lets a caller time / schedule the two halves separately). */
int hwy_highway_reset(const HwyHighwayParams *p, const HwyHighwayState *s, const HwyLinearTraffic *t,
                      const uint8_t *mask_a, const uint8_t *mask_b, float *obs, void *stream);

/* KinematicObservation.observe() (observation.py:234-276) for all envs. */
int hwy_highway_observe(const HwyHighwayParams *p, const HwyHighwayState *s, float *obs,
                        void *stream);

/* One AbstractEnv.step (abstract.py:259-285) for all envs: simulation_frequency //
 * policy_frequency substeps of {action_type.act on frame 0; Road.act; Road.step}, then
 * observe / _reward / _is_terminated / _is_truncated.
 *   action_i [n_envs] int32 (DiscreteMetaAction) or action_f [n_envs][2] float32
 *   (ContinuousAction); the unused one may be NULL.
 *   obs [n_envs][K][5] f32, reward [n_envs] f64, terminated/truncated [n_envs] u8.
 *   info_speed [n_envs] f64 / info_crashed [n_envs] u8 (either may be NULL): the ego's speed
 *   and crashed flag of AbstractEnv._info (abstract.py:200-217) at the end of the step,
 *   before any autoreset.
 *   autoreset = HWY_AUTORESET_SAME_STEP: envs that ended are reset from their RNG stream
 *   in the same call and `obs` holds the reset observation; `final_obs` (may be NULL)
 *   receives the pre-reset observation of every env. */
int hwy_highway_step(const HwyHighwayParams *p, const HwyHighwayState *s, const HwyLinearTraffic *t,
                     const int32_t *action_i, const float *action_f, float *obs, double *reward,
                     uint8_t *terminated, uint8_t *truncated, double *info_speed, uint8_t *info_crashed,
                     int autoreset, float *final_obs, void *stream);

/* The operator seam `_simulate` uses (envs/common/abstract.py:304-307 without action_type.act):
 * `n_substeps` times  Road.act()  (road/road.py:464-467)  then  Road.step(1 / simulation_frequency)  (:469-481)
 * on the stored state, and nothing else — no observation, reward, clock or reset.  The controlled vehicle acts like
 * ControlledVehicle.act(None) (its current target lane / speed); a ContinuousAction ego keeps the action dict given in
 * `action_f` ([n_envs, 2] in [-1, 1], as for hwy_highway_step) or the default {steering 0, acceleration 0} if NULL.
 * What BASELINE.md's "Road.act() + Road.step(dt)" timing runs. */
int hwy_highway_substeps(const HwyHighwayParams *p, const HwyHighwayState *s, const HwyLinearTraffic *t,
                         int n_substeps, const float *action_f, void *stream);

/* ====================================================================== general road networks
 * roundabout-v0 (envs/roundabout_env.py): Straight / Sine / Circular lanes (road/lane.py:159-384),
 * planned routes and RoadNetwork.next_lane (road/road.py:73-157), TimeToCollision or absolute
 * Kinematics observation.  Same conventions as the highway entry points above. */
#define HWY_NET_MAX_LANES 32
#define HWY_NET_MAX_NODES 64
#define HWY_NET_MAX_SUCC 6
#define HWY_NET_MAX_ROUTE 16
#define HWY_NET_GROUP 8        /* vehicle slots per env (threads per env): roundabout-v0 */
#define HWY_NET_GROUP_LARGE 32 /* intersection-v0 (dynamic population, at most 32 vehicles) */

#define HWY_LANE_STRAIGHT 0
#define HWY_LANE_SINE 1
#define HWY_LANE_CIRCULAR 2

#define HWY_OBS_KINEMATICS 0
#define HWY_OBS_OCCUPANCY 1 /* envs/common/observation.py:279-499, default 4 x 11 x 11 grid */
#define HWY_OBS_TTC 2

#define HWY_META_YIELDING (1 << 22)
#define HWY_META_NO_LANE_CHANGE (1 << 23) /* IDMVehicle(enable_lane_change=False) (vehicle/behavior.py:48-62,104-105) */ /* RegulatedRoad: vehicle.is_yielding (road/regulation.py:42-83) */

/* One lane of RoadNetwork.graph[from][to][lane_id]; table order = graph enumeration order
 * (road/road.py:65-71: from-node insertion order, to-node insertion order, lane id). */
typedef struct HwyNetLane {
    int32_t type, from_node, to_node, lane_id;
    int32_t road_first, road_count; /* table index of lane 0 of this road; lanes on the road */
    int32_t forbidden, priority;
    int32_t exit_lane, _pad; /* intersection: "il" in the from-node and "o" in the to-node name (intersection_env.py:354-373) */
    double width, speed_limit, length;
    double sx, sy, ex, ey, dx, dy, lx, ly, heading;            /* StraightLane / SineLane base */
    double amplitude, pulsation, phase;                         /* SineLane */
    double cx, cy, radius, start_phase, end_phase, direction;   /* CircularLane */
} HwyNetLane;

/* Device-resident, immutable after construction. */
typedef struct HwyNetGraph {
    int32_t n_lanes, n_nodes;
    HwyNetLane lanes[HWY_NET_MAX_LANES];
    int32_t succ_count[HWY_NET_MAX_NODES];            /* graph[node].keys() in insertion order: */
    int32_t succ[HWY_NET_MAX_NODES][HWY_NET_MAX_SUCC]; /* first-lane table index of each road   */
} HwyNetGraph;

typedef struct HwyNetParams {
    int32_t n_vehicles; /* <= HWY_NET_GROUP; slot 0 is the MDPVehicle ego */
    int32_t simulation_frequency, policy_frequency;
    int32_t n_target_speeds;
    int32_t obs_type;   /* HWY_OBS_* */
    int32_t obs_vehicles_count, obs_see_behind, obs_absolute, obs_normalize, obs_clip;
    int32_t ttc_horizon;
    int32_t normalize_reward;
    double duration;
    double target_speeds[HWY_MAX_TARGET_SPEEDS];
    double obs_x_lo, obs_x_hi, obs_y_lo, obs_y_hi, obs_vx_lo, obs_vx_hi, obs_vy_lo, obs_vy_hi;
    double collision_reward, high_speed_reward, lane_change_reward; /* roundabout_env.py:30-34 */
    double acc_max, comfort_acc_max, comfort_acc_min, distance_wanted, time_wanted;
    double politeness, lane_change_min_acc_gain, lane_change_max_braking_imposed, lane_change_delay;
    double perception_distance;
    /* intersection-v0 (envs/intersection_env.py) */
    int32_t regulated;          /* RegulatedRoad (road/regulation.py:12-111) */
    int32_t action_mode;        /* 0: LANE_LEFT/IDLE/LANE_RIGHT/FASTER/SLOWER; 1: SLOWER/IDLE/FASTER (action.py:204-206) */
    int32_t reward_type;        /* 0 roundabout_env.py:44-71, 1 intersection_env.py:79-117 */
    int32_t obs_features;       /* Kinematics columns: 5, or 7 with cos_h, sin_h */
    int32_t offroad_terminal;
    int32_t dynamic_population; /* per-step _clear_vehicles / _spawn_vehicle (intersection_env.py:136-140) */
    int32_t connected_lanes;    /* config["neighbour_vehicles_connected_lanes"]: roundabout-v1, intersection-v2
                                 * (abstract.py:26-37, road/road.py:509-529) */
    int32_t n_agents;           /* config["controlled_vehicles"] (0 or 1: one).  > 1 = MultiAgentAction /
                                 * MultiAgentObservation (action.py:301-333, observation.py:588-604): actions, obs and
                                 * speed_index carry n_agents entries per env, controlled vehicles in list order */
    double arrived_reward, reward_speed_lo, reward_speed_hi;
    /* merge-v0 (envs/merge_env.py:24-84): reward_type 2 */
    double right_lane_reward, merging_speed_reward;
    int32_t merge_lane;         /* table index of ("b", "c", 2): slow ControlledVehicles there are penalised; -1: none */
    int32_t merge_end_lane;     /* 0: terminated past x = 370 (merge-v0); > 0: table index of a ("c","d",k) lane,
                                 * terminated past its end x - 90 (MergeGenericEnv.end_position, merge_env.py:249) */
    double left_lane_reward;    /* two-way-v0 (envs/two_way_env.py:17-62): reward_type 3; u-turn-v0
                                 * (envs/u_turn_env.py:14-82): reward_type 4 */
    /* exit-v0 (envs/exit_env.py:147-198): reward_type 5 = collision, goal (the TARGET lane is ("1","2",lanes_count) or
     * ("2","exit",0)), clipped speed term, target lane id; normalised to [collision_reward, goal_reward], clipped */
    double goal_reward;
    int32_t exit_lane_a, exit_lane_b;
    int32_t obs_exit_lane;      /* ExitObservation (observation.py:624-675): table index (> 0) of ("1","2",-1), whose
                                 * longitudinal coordinate replaces x in the ego row of the Kinematics table; 0: none */
    int32_t _pad_exit;
    /* ContinuousAction / DiscreteAction on a network env (envs/common/action.py:73-196; intersection-v1): the
     * controlled vehicle is a plain Vehicle (kind HWY_KIND_VEHICLE) or, with `dynamical`, a BicycleVehicle
     * (vehicle/dynamics.py:33-160, whose lateral_speed / yaw_rate live in the vehicle's tt pair).  `action` of the
     * step entry points then points to float32 [n_envs][2] = (throttle, steering) in [-1, 1]. */
    int32_t action_type;        /* 0 DiscreteMetaAction labels (int32), 1 ContinuousAction (float32 pairs) */
    int32_t act_clip, dynamical;
    int32_t obs_n_feat;         /* > 0: Kinematics columns obs_feat[0..n) (HWY_FEAT_*, any Vehicle.to_dict key) with
                                 * per-column ranges; 0: the (presence, x, y, vx, vy [, cos_h, sin_h]) table above */
    double acc_lo, acc_hi, steer_lo, steer_hi;
    int32_t obs_feat[HWY_MAX_OBS_FEATURES], obs_feat_ranged[HWY_MAX_OBS_FEATURES];
    double obs_feat_lo[HWY_MAX_OBS_FEATURES], obs_feat_hi[HWY_MAX_OBS_FEATURES];
} HwyNetParams;

/* route entry: from_node | to_node << 8 | (lane_id + 1) << 16  (lane_id + 1 == 0: None) */
typedef struct HwyNetState {
    int32_t n_envs;
    int32_t vp;                  /* slot stride == HWY_NET_GROUP */
    double *pos, *hs, *tt, *imp; /* [n_envs*vp*2], as HwyHighwayState */
    double *delta;               /* [n_envs*vp] */
    int32_t *meta;               /* [n_envs*vp] lane(8) | target lane(8) | flags, as above */
    int32_t *route;              /* [n_envs*vp*HWY_NET_MAX_ROUTE] ControlledVehicle.route */
    int32_t *route_len;          /* [n_envs*vp] */
    int32_t *speed_index;        /* [n_envs * max(1, n_agents)] MDPVehicle.speed_index of each controlled vehicle */
    double *time;                /* [n_envs] */
    int32_t *count;              /* [n_envs] vehicles currently on the road; NULL: always n_vehicles */
    int32_t *road_steps;         /* [n_envs] RegulatedRoad.steps; NULL when not regulated */
    uint64_t *rng;               /* [5*n_envs] numpy PCG64 stream (layout as HwyHighwayState.rng); NULL if unused */
    double *reward_terms;        /* [n_envs*HWY_REWARD_TERMS] or NULL: un-weighted terms of _rewards (info["rewards"]) by
                                  * reward_type: 0 roundabout {collision, high_speed, lane_change, on_road}; 1 intersection
                                  * {collision, high_speed, arrived, on_road} (mean over the agents); 2 merge {collision,
                                  * right_lane, high_speed, lane_change, merging_speed}; 3 two-way {high_speed, left_lane};
                                  * 4 u-turn {collision, left_lane, high_speed, on_road} */
    int32_t *overflow;           /* [n_envs] or NULL: vehicles that _spawn_vehicle accepted but that found every slot of
                                  * the env taken (the reference's list is unbounded; HWY_NET_GROUP_LARGE slots here).
                                  * Incremented by the step / reset kernels, never cleared by them: a non-zero entry
                                  * means the env has left the reference's trajectory (info["spawn_overflow"]) */
} HwyNetState;

/* intersection-v0 (HWY_SCENARIO_INTERSECTION, s->vp == HWY_NET_GROUP_LARGE).
 * Step: RegulatedRoad rules every int(simulation_frequency / 2) substeps, and after the observation the step's
 * _clear_vehicles and _spawn_vehicle(spawn_probability) drawing from s->rng (IntersectionEnv.step, :136-140), with
 * these _spawn_vehicle constants (envs/intersection_env.py:325-352).  With config["controlled_vehicles"] =
 * p->n_agents > 1 (intersection-multi-agent-v0, envs/intersection_env.py:376-420): action [n_envs][n_agents], obs
 * [n_envs][n_agents][K][F]; reward is the mean of the agents' rewards, terminated = any crashed or all arrived
 * (:62-134); agents_reward / agents_terminated [n_envs][n_agents] (NULL for a single agent; optional) are _info's
 * per-agent entries, which MultiAgentWrapper (abstract.py:468-477) returns in place of the scalar reward / terminated.
 * Reset: IntersectionEnv._reset / _make_vehicles (:119-122,245-323): n-1 _spawn_vehicle draws, 3 s of warm-up
 * simulation, the challenger, the controlled vehicle (MDPVehicle on ("o0","ir0",0) at 60 + 5*normal(1)), the 20 m
 * pruning; all draws come from s->rng in the reference's order. */
typedef struct HwyIntersectionSpawn {
    int32_t spawn_lane[4];      /* table index of ("o"+k, "ir"+k, 0) */
    double spawn_probability;   /* config["spawn_probability"] */
    const int32_t *route_table; /* DEVICE [n_lanes][4][HWY_NET_MAX_ROUTE]: plan_route_to(lane, "o"+k) */
    const int32_t *route_len;   /* DEVICE [n_lanes][4] */
    /* _make_vehicles (:245-323), used by the reset */
    int32_t ego_lane;              /* table index of ("o0", "ir0", 0) */
    int32_t ego_destination;       /* k of config["destination"] == "o"+k; -1 (None): "o" + integers(1, 4) */
    int32_t initial_vehicle_count; /* config["initial_vehicle_count"] */
    int32_t _pad;
    int32_t *scratch;              /* DEVICE [2 * (n_envs + 1)] int32: work lists (envs being reset; the
                                    * step's 16-slot / 32-slot populations).  NULL: the step runs every env
                                    * on 32 slots and the reset is unavailable */
} HwyIntersectionSpawn;

/* observation size in floats PER ENV: Kinematics K*F, TimeToCollision 3*3*(horizon*policy_frequency),
 * OccupancyGrid 4*11*11; times n_agents when several vehicles are controlled */
int hwy_network_obs_size(const HwyNetParams *p);

/* Test entries (the reference's own known-answer tests run against the device functions):
 * Road.neighbour_vehicles(v, lane) (road/road.py:483-547) for every vehicle v of every env — lane = query_lane
 * [n_envs*vp] or, when NULL, v's own lane — into front / rear [n_envs*vp] (slot index, -1 = None);
 * utils.rotated_rectangles_intersect (utils.py:115-125) for n pairs, rects [n][10] =
 * (cx, cy, length, width, angle) x 2 on the DEVICE. */
int hwy_debug_network_neighbours(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetState *s,
                                 const int32_t *query_lane, int32_t *front, int32_t *rear, void *stream);
int hwy_debug_rotated_rectangles_intersect(const double *rects, int n, int32_t *out, void *stream);

/* The lane functions of the network kernels (csrc/hwy_lanes.cuh) on n inputs, one thread each, on the lane table as
 * the kernels stage it (the arcs' end points in sx, sy, ex, ey).  graph is a HOST pointer (1..HWY_NET_MAX_LANES
 * lanes); in [n][HWY_LANES_IN] and out [n][k_out] are DEVICE doubles, in[0] the table index of the lane:
 *   LOCAL lane, x, y -> s, lat (lane_local)               POSITION lane, s, lat -> x, y (lane_position)
 *   HEADING_AT lane, s -> heading (lane_heading_at)
 *   DISTANCE_WITH_HEADING lane, x, y, h -> d, s, lat (lane_distance_with_heading)
 *   ON lane, x, y -> 1 / 0: lane_local, then lane_on(margin = 1)
 *   MAYBE_ON lane, x, y -> 1 / 0: lane_maybe_on, the neighbour search's pre-test of ON
 *   PRUNABLE lane, x, y, bd -> 1 / 0: closest_lane_prunable with a fresh circle cache
 *   PRUNABLE_SCAN hint, x, y, bd -> [HWY_NET_MAX_LANES] closest_lane_prunable of every lane in table order with one
 *                 circle cache carried across them, the hint skipped, as closest_lane_group scans (0 for the hint and
 *                 past the table's end)
 * An in[0] that is not a lane of the table gives NaN outputs. */
#define HWY_LANES_IN 5
enum {
    HWY_LANES_LOCAL = 0, HWY_LANES_POSITION, HWY_LANES_HEADING_AT, HWY_LANES_DISTANCE_WITH_HEADING, HWY_LANES_ON,
    HWY_LANES_MAYBE_ON, HWY_LANES_PRUNABLE, HWY_LANES_PRUNABLE_SCAN
};
int hwy_debug_network_lanes(const HwyNetGraph *graph, int op, const double *in, double *out, int n, void *stream);
/* Vehicle.on_state_update's closest-lane search (closest_lane_group) of every vehicle of every env, the lane in each
 * vehicle's meta word as the search's starting lane: lane [n_envs*vp] (-1 past the env's count), own_s / own_lat
 * [n_envs*vp] its local coordinates on that lane.  graph is a DEVICE pointer, as for the step entry points. */
int hwy_debug_network_closest_lanes(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetState *s,
                                    int32_t *lane, double *own_s, double *own_lat, void *stream);

/* The scalar device functions of the step kernels (csrc/hwy_math.cuh, csrc/hwy_device.cuh) on n inputs, one thread
 * each: in [n][k_in] and out [n][k_out] are DEVICE doubles; the operands of each op, in order, are
 *   SINCOS x -> sin, cos (m_sincos)          IDM_POW x, delta -> x ** delta     EXP_DLOG d, x -> exp(d log x)
 *   PY_MOD_POS a, b -> a % b (b > 0)         WRAP_TO_PI x                        NOT_ZERO x
 *   DIV_FINITE n, d -> n / d                 DOT2 a0, a1, b0, b1 -> np.dot       NORM2 a0, a1 -> np.linalg.norm
 *   BETA_CONTROLLED x -> sin, cos of the slip angle for the steering sine x (beta_of_controlled)
 *   BETA_ANGLE delta -> sin, cos of arctan(tan(delta) / 2)
 *   SPEED_TO_INDEX speed, n_target_speeds, target_speeds[HWY_MAX_TARGET_SPEEDS] -> index (as a double); NaN when
 *                  n_target_speeds is not in 1..HWY_MAX_TARGET_SPEEDS. */
enum {
    HWY_MATH_SINCOS = 0, HWY_MATH_IDM_POW, HWY_MATH_EXP_DLOG, HWY_MATH_PY_MOD_POS, HWY_MATH_WRAP_TO_PI,
    HWY_MATH_NOT_ZERO, HWY_MATH_DIV_FINITE, HWY_MATH_DOT2, HWY_MATH_NORM2, HWY_MATH_BETA_CONTROLLED,
    HWY_MATH_BETA_ANGLE, HWY_MATH_SPEED_TO_INDEX
};
int hwy_debug_math(int op, const double *in, double *out, int n, void *stream);

/* The numpy Generator(PCG64) restatement of the kernels, one generator per thread: words_in / words_out [5][n] in
 * the HwyHighwayState.rng layout (DEVICE).  Each thread makes `count` draws of kind op into draws [n][count]
 * (uint64; doubles as their IEEE bits): NEXT64, NEXT32, NEXT_DOUBLE, UNIFORM(arg_lo, arg_hi), CHOICE(arg_i) and
 * NORMAL, which writes [n][count][2] = (value bits, 64-bit outputs the draw consumed; 0 when more than 16), then
 * stores its generator in words_out.  AT positions the generator at output arg_i of its stream (the jump table of
 * the fused autoreset, 0 <= arg_i < 4 * HWY_MAX_VEHICLES + 8) and draws nothing. */
enum {
    HWY_PCG_NEXT64 = 0, HWY_PCG_NEXT32, HWY_PCG_NEXT_DOUBLE, HWY_PCG_UNIFORM, HWY_PCG_NORMAL, HWY_PCG_CHOICE,
    HWY_PCG_AT
};
int hwy_debug_pcg64(int op, int arg_i, double arg_lo, double arg_hi, int count, const uint64_t *words_in,
                    uint64_t *words_out, uint64_t *draws, int n, void *stream);

/* observation_type.observe() of the current state */
int hwy_network_observe(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetState *s,
                        float *obs, void *stream);

/* merge-v0 (HWY_SCENARIO_MERGE): MergeEnv._make_vehicles + the Obstacle of _make_road (envs/merge_env.py:150-190)
 * on the device: the MDPVehicle on ("a","b",1) at s = 30, speed 30; three IDM vehicles on ("a","b", integers(2)) at
 * position + uniform(-5, 5) with speed + uniform(-1, 1); the merging vehicle on ("j","k",0) at s = 110, speed 20,
 * target speed 30; and, in the slot after the vehicles, the Obstacle (kind HWY_KIND_OBSTACLE) at the end of the
 * ramp. */
typedef struct HwyMergeSpawn {
    int32_t lane_ab[2];      /* table indices of ("a","b",0), ("a","b",1) */
    int32_t lane_jk;         /* ("j","k",0) */
    int32_t ego_speed_index; /* MDPVehicle.speed_to_index(30) */
    double obstacle_x, obstacle_y;
    /* merge-generic-v0 / v1 (MergeGenericEnv._make_vehicles, envs/merge_env.py:320-368) when lanes_count > 0: the
     * MDPVehicle on ("a","b",lanes_count-1) at s = 30, speed 30; then for each of vehicles_count vehicles up to 10
     * tries of integers(lanes_count) (no draw for one lane) and uniform(0, max_position), rejected unless the
     * longitudinal lies more than 15 m from every one already placed on that lane id (the ego's 30 included); an
     * accepted try draws its speed 30 + uniform(-2, 2) and is placed at ("a","b",k).position(s, 0), which may lie past
     * the lane's end.  Then the merging IDM vehicle on ("j","k",0) at s = 60, speed 20, target speed 30, and the
     * Obstacle last.  Every object takes its closest lane at heading 0.  Lane k of ("a","b") is lane_ab[0] + k.  A
     * vehicle whose 10 tries fail is skipped: s->count (required) receives the population (the Obstacle's slot is
     * count - 1) and the slots past it are cleared.  Slot stride 8 or 32; on 32 slots the step is the one without
     * rules or population changes.  This tail grew the struct from 32 to 48 bytes inside the union, whose size and
     * offset did not change (the union's largest member is HwyUTurnSpawn). */
    int32_t lanes_count;     /* config["lanes_count"], 1..9; 0: merge-v0's fixed placement above */
    int32_t vehicles_count;  /* config["vehicles_count"], at most s->vp - 3 (<= 0: no traffic) */
    double max_position;     /* before + converge + parallel merge lengths, the traffic's uniform upper bound */
} HwyMergeSpawn;

/* u-turn-v0 (HWY_SCENARIO_U_TURN): UTurnEnv._make_vehicles (envs/u_turn_env.py:179-275) on the device: the
 * MDPVehicle at the start of ("a","b",0), speed 16, and six IDM vehicles made with make_on_lane(lane[v],
 * longitudinal[v] + 2 normal(), speed[v] + 2 normal()); vehicle 1 also draws its DELTA (randomize_behavior); every
 * vehicle gets plan_route_to("d") from a host-built table indexed by the closest lane.  (The reference also sets
 * ego.PURSUIT_TAU, an attribute nothing reads — steering_control uses TAU_PURSUIT, vehicle/controller.py:28,159 — so
 * there is nothing to restate.) */
typedef struct HwyUTurnSpawn {
    int32_t lane[8];             /* [0] ego lane ("a","b",0); [1..6] make_on_lane lanes */
    double longitudinal[8], speed[8];
    int32_t ego_speed_index, _pad;
    const int32_t *route_table;  /* DEVICE [n_lanes][HWY_NET_MAX_ROUTE]: plan_route_to("d") from each lane */
    const int32_t *route_len;    /* DEVICE [n_lanes] */
} HwyUTurnSpawn;

/* exit-v0 (HWY_SCENARIO_EXIT): ExitEnv._create_vehicles (envs/exit_env.py:107-145) on the device: the MDPVehicle from
 * Vehicle.create_random(speed=25, lane ("0","1",0), spacing=ego_spacing); vehicles_count IDMVehicles on ("0","1",
 * choice(lanes, p=lanes/sum)) at the lane's speed limit, spacing 1 / vehicles_density, routed to "3",
 * enable_lane_change=False.  State stride 32, s->count is set to n_vehicles.  The step is the 32-slot one without
 * rules or population changes. */
typedef struct HwyExitSpawn {
    int32_t lanes_count, n_vehicles;   /* config["lanes_count"], 1 + config["vehicles_count"] */
    int32_t ego_speed_index, _pad;
    double ego_speed, ego_spacing, vehicles_density;
    double spawn_exp;                  /* np.exp(-5 / 40 * lanes_count) (vehicle/kinematics.py:95) */
    double cdf[HWY_MAX_LANES];         /* Generator.choice(p=lanes / lanes.sum()): p.cumsum() / cumsum[-1] */
    int32_t route_12, route_23;        /* encoded route entries ("1","2",None), ("2","3",None) */
} HwyExitSpawn;

/* two-way-v0 (HWY_SCENARIO_TWO_WAY): TwoWayEnv._make_vehicles (envs/two_way_env.py:113-158) on the device: the
 * MDPVehicle on ("a","b",1) at s = 30, three IDM vehicles ahead at 70 + 40 i + 10 normal() with speed 24 + 2 normal(),
 * two oncoming ones on ("b","a",0) at 200 + 100 i + 10 normal() with speed 20 + 5 normal(); all traffic has
 * enable_lane_change=False. */
typedef struct HwyTwoWaySpawn {
    int32_t lane_ab1, lane_ba0; /* table indices of ("a","b",1) and ("b","a",0) */
    int32_t ego_speed_index, _pad;
} HwyTwoWaySpawn;

/* roundabout-v0 (HWY_SCENARIO_ROUNDABOUT): RoundaboutEnv._make_vehicles (envs/roundabout_env.py:317-391) on the
 * device.  Per traffic vehicle the env's numpy stream yields normal (longitudinal), normal (speed),
 * choice(destinations), uniform (DELTA); routes come from a host-built table of ControlledVehicle.plan_route_to
 * results (vehicle/controller.py:71-87). */
typedef struct HwyRoundaboutSpawn {
    int32_t ego_lane;            /* table index of ("ser", "ses", 0) */
    int32_t spawn_lane[4];       /* make_on_lane lanes: (we,sx,1), (we,sx,0), (we,sx,0), (eer,ees,0) */
    int32_t fixed_destination;   /* config["incoming_vehicle_destination"], -1 = None */
    int32_t ego_speed_index;
    int32_t _pad;
    double base_longitudinal[4]; /* 5, 20, -20, 50 */
    double ego_longitudinal, ego_heading_longitudinal, ego_speed; /* 125, 140, 8 */
    double position_deviation, speed_deviation, traffic_speed;    /* 2, 2, 16 */
    double delta_lo, delta_hi;   /* IDMVehicle.DELTA_RANGE */
    const int32_t *route_table;  /* DEVICE [n_lanes][4][HWY_NET_MAX_ROUTE]; destination 0..2 = exr, sxr, nxr; 3 = the ego's nxs */
    const int32_t *route_len;    /* DEVICE [n_lanes][4] */
} HwyRoundaboutSpawn;

/* roundabout-generic-v0 / v1 (HWY_SCENARIO_ROUNDABOUT_GENERIC): RoundaboutGenericEnv._make_vehicles
 * (envs/roundabout_env.py:664-751) on the device: the MDPVehicle at length - 2.5 of ("ser","ses",0), speed 8, routed
 * to "nxs"; then for each of vehicles_count vehicles up to 10 tries of integers(0, 7) (spawn road), integers(0, lanes
 * of the road) (no draw on a one-lane road), uniform(5, max(5, length - 5)) (longitudinal), rejected when the point
 * lies closer than 7 m to a point already placed; an accepted try draws its speed 14 + 2 normal(), its destination
 * integers(0, 4) (none when fixed_destination >= 0) and DELTA uniform(3.5, 4.5), and plans its route from its closest
 * lane.  A vehicle whose 10 tries all fail is skipped: s->count (required) receives the population and the slots past
 * it are cleared.  Slot stride 8 or 32; on 32 slots the step is the one without rules or population changes. */
typedef struct HwyRoundaboutGenericSpawn {
    int32_t ego_lane;            /* table index of ("ser", "ses", 0) */
    int32_t spawn_road[7];       /* table index of lane 0 of (we,sx), (sx,se), (ee,nx), (nx,ne), (eer,ees), (ner,nes),
                                  * (wer,wes) */
    int32_t vehicles_count;      /* config["vehicles_count"], at most s->vp - 1 (<= 0: the ego alone) */
    int32_t fixed_destination;   /* destinations[min(incoming_vehicle_destination, 3)] as 0..3; -1 = None (drawn) */
    int32_t ego_speed_index;     /* MDPVehicle.speed_to_index(8) */
    int32_t route_width;         /* destinations per lane of the route table, >= 5 */
    const int32_t *route_table;  /* DEVICE [n_lanes][route_width][HWY_NET_MAX_ROUTE]; destination 0..3 = exr, sxr,
                                  * nxr, wxr; 4 = the ego's nxs */
    const int32_t *route_len;    /* DEVICE [n_lanes][route_width] */
} HwyRoundaboutGenericSpawn;

/* racetrack-v0 / v1 and racetrack-large / racetrack-oval (HWY_SCENARIO_RACETRACK): RacetrackEnv
 * (envs/racetrack_env.py:15-425; v1 with connected_lanes) and its large (RacetrackEnvLarge, :432-880) and oval
 * (RacetrackEnvOval, :882-1396) tracks on the 8-slot network state, which must carry s->count (the population: the
 * ego, the front vehicle and the extra vehicles that survived the 20 m check).  The controlled vehicle is a plain
 * Vehicle (HWY_KIND_VEHICLE) in slot 0 whose (target_speed, timer) pair holds its persisting action dict
 * (acceleration, steering) (vehicle/kinematics.py:119-128); `action` is float32 [n_envs][2] = (throttle, steering) as
 * passed, a missing control axis staged as 0 with the range (0, 0) in p.
 * Reset: _make_vehicles (:374-425), drawing from s->rng in the reference's order; slots past the population are
 * cleared.  Step: one RacetrackEnv.step of every env — the action, simulation_frequency / policy_frequency substeps,
 * observation, reward (:66-83; s->reward_terms: lane_centering, action, collision, on_road), terminated (crashed, or
 * off road with terminate_off_road), truncated (time >= duration).  Substeps: Road.act + Road.step with the
 * persisting action, on every env. */
typedef struct HwyRacetrackParams {
    int32_t other_vehicles;      /* config["other_vehicles"], 0..HWY_NET_GROUP - 1 */
    int32_t terminate_off_road;  /* config["terminate_off_road"] */
    int32_t lane_ab, lane_bc;    /* table index of ("a","b",0) and ("b","c",0) */
    int32_t n_from_nodes;        /* len(network.graph): random_lane_index draws among nodes 0 .. n-1 */
    int32_t ego_lanes;           /* the ego's lane draw integers(ego_lanes): 2 (racetrack, large), no_lanes (oval);
                                  * at most the lane count of ("a","b") and of ("b","c"), which the caller checks */
    double lane_centering_cost, lane_centering_reward, action_reward, collision_reward, on_road_reward;
} HwyRacetrackParams;

/* The scenario of a network entry point: `kind` names the union member the entry reads.  HWY_SCENARIO_NONE (or a NULL
 * scenario where one is optional) reads none: the step and the substeps then run the plain network kernels. */
enum {
    HWY_SCENARIO_NONE = 0, HWY_SCENARIO_ROUNDABOUT, HWY_SCENARIO_ROUNDABOUT_GENERIC, HWY_SCENARIO_MERGE,
    HWY_SCENARIO_TWO_WAY, HWY_SCENARIO_U_TURN, HWY_SCENARIO_EXIT, HWY_SCENARIO_INTERSECTION, HWY_SCENARIO_RACETRACK
};
typedef struct HwyNetScenario {
    int32_t kind, _pad; /* HWY_SCENARIO_* */
    union {
        HwyRoundaboutSpawn roundabout;
        HwyRoundaboutGenericSpawn roundabout_generic;
        HwyMergeSpawn merge;
        HwyTwoWaySpawn two_way;
        HwyUTurnSpawn u_turn;
        HwyExitSpawn exit;
        HwyIntersectionSpawn intersection;
        HwyRacetrackParams racetrack;
    } u;
} HwyNetScenario;

/* AbstractEnv.reset()'s _reset() of scenario sc (required, not NONE) for the envs with mask_a[e] | mask_b[e] (both
 * NULL: every env), drawing from s->rng (required).  With final_obs, obs is first copied there (the SameStep
 * autoreset's info["final_obs"]); with obs, the fresh observation of the reset envs is written to obs. */
int hwy_network_reset(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetScenario *sc, const HwyNetState *s,
                      const uint8_t *mask_a, const uint8_t *mask_b, float *obs, float *final_obs, void *stream);

/* AbstractEnv.step (abstract.py:259-285) of every env on a general network.  graph is a DEVICE pointer; sc may be
 * NULL (kind NONE).  action: int32 DiscreteMetaAction labels (action.py:204), [n_envs] or [n_envs][n_agents]; float32
 * [n_envs][2] (throttle, steering) when p->action_type == 1.  obs [n_envs][hwy_network_obs_size] f32, reward [n_envs]
 * f64, terminated / truncated [n_envs] u8; info_speed [n_envs] f64 / info_crashed [n_envs] u8 (either may be NULL);
 * agents_reward / agents_terminated: see HwyIntersectionSpawn.  Kind RACETRACK runs the racetrack step; every other
 * kind runs on the slot stride: 8 slots the roundabout family's step, 32 slots the intersection family's, with the
 * rules, population changes and 16 / 32-slot split of kind INTERSECTION, without them for any other kind. */
int hwy_network_step(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetScenario *sc, const HwyNetState *s,
                     const void *action, float *obs, double *reward, uint8_t *terminated, uint8_t *truncated,
                     double *info_speed, uint8_t *info_crashed, double *agents_reward, uint8_t *agents_terminated,
                     void *stream);

/* Road.act() + Road.step(dt) n_substeps times without an ego action, and nothing else, for the envs whose mask byte
 * is set (NULL: all): the 3 s warm-up of IntersectionEnv._make_vehicles (:271-278), and env.road_substeps.  sc may be
 * NULL (kind NONE).  Kind RACETRACK runs every env (mask must be NULL), its plain ego keeping its persisting action;
 * there n_substeps == 0 launches nothing. */
int hwy_network_substeps(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetScenario *sc,
                         const HwyNetState *s, const uint8_t *mask, int n_substeps, void *stream);

/* ====================================================================== observation plugins on ANY road family
 * The reference's observation_factory (envs/common/observation.py:772-794) builds any ObservationType on any env; these
 * entry points are that registry on the device: they read a state of either family through a HwyObsView (the highway
 * family passes the lane table of RoadNetwork.straight_road_network as a HwyNetGraph) and write the observation of
 * every controlled vehicle, obs[n_envs][max(1, n_agents)][...].  mask_a | mask_b select envs (both NULL: all). */
#define HWY_FEAT_ON_ROAD 13 /* OccupancyGrid layer (observation.py:412-413) */
#define HWY_FEAT_UNKNOWN 14 /* a feature no Vehicle.to_dict key matches: the layer stays NaN -> 0 */

typedef struct HwyObsView {
    int32_t n_envs, vp;         /* slot stride of the state arrays */
    int32_t n_vehicles;         /* slots in use when count == NULL */
    int32_t n_agents;           /* controlled vehicles observed per env (0 or 1: the first one) */
    const double *pos, *hs;     /* [n_envs*vp*2] position, (heading, speed) */
    const int32_t *meta;        /* [n_envs*vp] lane | kind | ... (HWY_META_*) */
    const int32_t *count;       /* [n_envs] or NULL */
    const int32_t *route;       /* [n_envs*vp*HWY_NET_MAX_ROUTE] or NULL (no planned routes: cos_d = sin_d = 0) */
    const int32_t *route_len;   /* [n_envs*vp] or NULL */
    const int32_t *speed_index; /* [n_envs*max(1, n_agents)] MDPVehicle.speed_index (TimeToCollision) or NULL */
} HwyObsView;

/* OccupancyGridObservation.__init__ (observation.py:286-333) */
typedef struct HwyGridParams {
    int32_t n_features;
    int32_t features[HWY_MAX_OBS_FEATURES];  /* HWY_FEAT_* */
    int32_t ranged[HWY_MAX_OBS_FEATURES];    /* the feature has a features_range entry: lmap to [-1, 1] */
    double range_lo[HWY_MAX_OBS_FEATURES], range_hi[HWY_MAX_OBS_FEATURES];
    int32_t x_ranged, y_ranged;              /* "x" / "y" in features_range (cell index un-maps them, :383-400) */
    double x_lo, x_hi, y_lo, y_hi;
    double grid_lo[2], grid_step[2];
    int32_t shape[2];                        /* floor((grid_size[:,1] - grid_size[:,0]) / grid_step) */
    int32_t align_to_vehicle_axes, clip, as_image, observe_intentions;
} HwyGridParams;
/* obs [n_envs][agents][n_features][shape0][shape1] float32 (as_image: the uint8 values as floats) */
int hwy_observe_grid(const HwyNetGraph *graph, const HwyObsView *view, const HwyGridParams *p, const uint8_t *mask_a,
                     const uint8_t *mask_b, float *obs, void *stream);

/* TimeToCollisionObservation (observation.py:115-152; finite_mdp.py:104-163 compute_ttc_grid): obs
 * [n_envs][agents][3][3][horizon * policy_frequency] */
typedef struct HwyTtcParams {
    int32_t horizon, policy_frequency, n_target_speeds, _pad;
    double target_speeds[HWY_MAX_TARGET_SPEEDS];
} HwyTtcParams;
int hwy_observe_ttc(const HwyNetGraph *graph, const HwyObsView *view, const HwyTtcParams *p, const uint8_t *mask_a,
                    const uint8_t *mask_b, float *obs, void *stream);

/* AbstractEnv.to_finite_mdp() = finite_mdp(env, time_quantization=1 / policy_frequency, horizon)
 * (envs/common/abstract.py:452-453, envs/common/finite_mdp.py:17-203) of every env (one controlled vehicle, an
 * MDPVehicle with 5 DiscreteMetaAction actions).  With V = n_target_speeds, L_e = lanes of the ego's road,
 * T = n_t = int(horizon / (1 / policy_frequency)) and S_max = V * l_max * T (l_max >= every road's lane count):
 *   grid [n_envs][V][l_max][T] f64 compute_ttc_grid (lanes >= L_e: 0);  n_lanes, n_states [n_envs] i32 (L_e, V*L_e*T);
 *   state [n_envs] i64 ravel_multi_index((speed_index, lane_index[2], 0), (V, L_e, T));
 *   transition [n_envs][S_max][5] i32, reward [n_envs][S_max][5] f64, terminal [n_envs][S_max] u8, raveled in each
 *   env's own (V, L_e, T) shape; rows s >= n_states are self-loops with reward 0, terminal. */
typedef struct HwyFiniteMdpParams {
    int32_t policy_frequency, n_target_speeds;
    int32_t l_max, n_t;
    double horizon;
    double target_speeds[HWY_MAX_TARGET_SPEEDS];
    double collision_reward, right_lane_reward, high_speed_reward, lane_change_reward;
} HwyFiniteMdpParams;
int hwy_finite_mdp(const HwyNetGraph *graph, const HwyObsView *view, const HwyFiniteMdpParams *p, double *grid,
                   int32_t *n_lanes, int32_t *n_states, int64_t *state, int32_t *transition, double *reward,
                   uint8_t *terminal, void *stream);

/* Value iteration of n_envs deterministic MDPs (the semantics of rl-agents' ValueIterationAgent), one block per
 * env: Q_0 = 0; Q_new = reward + gamma * (terminal[s] ? 0 : max_a Q_k[transition[s, a]]); stop at the first k with
 * np.allclose(Q_k, Q_new) over the env's n_states rows (keeping Q_k) or after `iterations` updates.
 * transition [n_envs][s_max][n_actions] i32, reward f64, terminal [n_envs][s_max] u8, n_states [n_envs] i32;
 * q [n_envs][s_max][n_actions] f64 (rows >= n_states: 0), iterations_done [n_envs] i32 = updates in q, or -1 when
 * n_states is outside 0..s_max or a successor is outside 0..n_states-1 (q then stays 0).  With state [n_envs] i64
 * and action [n_envs] i64 (both or neither), action[e] = the first argmax of q[e][state[e]] (-1 when the env
 * failed or state is out of range).  s_max <= HWY_VI_MAX_STATES, n_actions <= HWY_VI_MAX_ACTIONS. */
#define HWY_VI_MAX_STATES 4096
#define HWY_VI_MAX_ACTIONS 8
typedef struct HwyValueIterationParams {
    int32_t n_envs, s_max, n_actions, iterations;
    double gamma;
    const int64_t *state; /* DEVICE or NULL */
    int64_t *action;      /* DEVICE or NULL */
} HwyValueIterationParams;
int hwy_value_iteration(const HwyValueIterationParams *p, const int32_t *transition, const double *reward,
                        const uint8_t *terminal, const int32_t *n_states, double *q, int32_t *iterations_done,
                        void *stream);

/* LidarObservation (observation.py:678-769): obs [n_envs][agents][cells][2] float32 (distance, relative radial speed) */
typedef struct HwyLidarParams {
    int32_t cells, normalize;
    double maximum_range;
} HwyLidarParams;
int hwy_observe_lidar(const HwyObsView *view, const HwyLidarParams *p, const uint8_t *mask_a, const uint8_t *mask_b,
                      float *obs, void *stream);

/* ====================================================================== env cloning and tree search
 * Row copies between the per-env buffers of two env instances (or within one): for every pair k and every buffer b,
 * bytes [dst[k] * row_bytes, (dst[k] + 1) * row_bytes) of bufs[b].dst take those of row src[k] of bufs[b].src.  One
 * launch for all buffers; 16-byte vector copies where both rows and row_bytes are 16-byte aligned, 4-byte copies where
 * they are 4-byte aligned, bytes otherwise.  dst [n_pairs], src [n_pairs] are DEVICE int64 row indices; the caller
 * guarantees they are in range, that dst has no duplicates and that no row is both read and written. */
#define HWY_COPY_MAX_BUFS 32
typedef struct HwyRowCopy {
    const void *src; /* DEVICE row 0 of the source buffer */
    void *dst;       /* DEVICE row 0 of the destination buffer */
    int64_t row_bytes;
} HwyRowCopy;
int hwy_copy_env_rows(const HwyRowCopy *bufs, int n_bufs, const int64_t *dst, const int64_t *src, int n_pairs,
                      void *stream);

/* DiscreteMetaAction.get_available_actions (envs/common/action.py:262-298) of the first controlled vehicle of every
 * env on a lane table: mask [n_envs][5] u8 over (LANE_LEFT, IDLE, LANE_RIGHT, FASTER, SLOWER).  A side lane (id - 1,
 * id + 1 on the ego's road, road/road.py:200-211) is available when it is_reachable_from the ego's position
 * (road/lane.py:104-118); FASTER / SLOWER unless speed_index sits at the end of the n_target_speeds. */
int hwy_available_actions(const HwyNetGraph *graph, const HwyObsView *view, int n_target_speeds, uint8_t *mask,
                          void *stream);

/* Optimistic deterministic planning (Hren & Munos 2008) over n_roots trees of max_nodes = 1 + 5 * expansions nodes,
 * [n_roots][max_nodes] arrays, node 0 the root.  Expansion k creates the children of the selected leaf at nodes
 * 1 + 5 k + a.  discount[d] = gamma^d and bound[d] = gamma^d / (1 - gamma) for d in 0..expansions + 1. */
typedef struct HwyOpdTree {
    int32_t n_roots, max_nodes, expansions, n_actions;
    const double *discount, *bound;           /* DEVICE [expansions + 2] */
    uint8_t *exists, *expanded, *terminal;    /* DEVICE [n_roots][max_nodes] */
    int32_t *parent, *action, *depth, *branch; /* DEVICE [n_roots][max_nodes]; branch = the root child's action */
    double *reward, *value, *upper;           /* DEVICE [n_roots][max_nodes] */
    int32_t *selected;                        /* DEVICE [n_roots][expansions]: the expanded leaf, -1 when none was open */
    int64_t *leaf_row;                        /* DEVICE [n_roots * n_actions]: store row of the leaf each work row copies */
    int64_t *recommended;                     /* DEVICE [n_roots] */
} HwyOpdTree;
/* Expansion k: (k == 0: reset every tree to its root) select, per root, the open leaf (exists, not expanded, not
 * terminal) with the largest upper bound, the lowest node on ties; write selected[:, k] and leaf_row[r * n_actions + a]
 * = r * max_nodes + leaf (the root itself when no leaf is open). */
int hwy_opd_select(const HwyOpdTree *t, int k, void *stream);
/* Record the children of expansion k from the work rows r * n_actions + a: available [.][n_actions] u8 (of the leaf's
 * state), reward f64, terminated / truncated u8 of the step that made them. */
int hwy_opd_record(const HwyOpdTree *t, int k, const uint8_t *available, const double *reward,
                   const uint8_t *terminated, const uint8_t *truncated, void *stream);
/* recommended[r] = the root child action whose subtree holds the largest value (the lowest action on ties). */
int hwy_opd_recommend(const HwyOpdTree *t, void *stream);

/* Open-loop Monte-Carlo tree search (rl-agents' MCTSAgent; the statement is tests/mcts_spec.py) over n_roots trees of
 * max_nodes = 1 + 5 * k slots, [n_roots][max_nodes] arrays, node 0 the root.  Expanding node p takes the 5 slots
 * child_base[p] + a at n_nodes.  A work env of n_roots rows re-simulates each episode from the root states; the
 * walk_* arrays carry each root's episode between the horizon's steps. */
typedef struct HwyMctsTree {
    int32_t n_roots, max_nodes, episodes, horizon;
    double temperature;
    uint64_t seed;
    const double *discount;                  /* DEVICE [horizon]: gamma^h */
    int64_t *decision;                       /* DEVICE [1]: act() calls so far, a key of every draw */
    uint8_t *exists, *expanded;              /* DEVICE [n_roots][max_nodes] */
    int32_t *parent, *action, *child_base, *n_children, *count; /* DEVICE [n_roots][max_nodes] */
    double *prior, *value;                   /* DEVICE [n_roots][max_nodes] */
    int32_t *n_nodes, *skipped;              /* DEVICE [n_roots]: slots in use; expansions skipped for lack of room */
    int32_t *walk_node;                      /* DEVICE [n_roots] */
    double *walk_return;                     /* DEVICE [n_roots] */
    uint8_t *walk_flags;                     /* DEVICE [n_roots]: bit 0 done, bit 1 rolling out */
    int32_t *leaf;                           /* DEVICE [n_roots][episodes]: the node each episode backed up from */
    double *returns;                         /* DEVICE [n_roots][episodes] */
    int32_t *remap;                          /* DEVICE [n_roots][max_nodes]: scratch of hwy_mcts_reroot */
    int32_t *actions;                        /* DEVICE [n_roots]: the work rows' next actions */
    int64_t *recommended;                    /* DEVICE [n_roots] */
} HwyMctsTree;
/* Step d of episode e: (d > 0) add the work rows' previous reward, terminated, truncated (u8 / f64 [n_roots]) to each
 * walk, then descend, expand (over available [n_roots][5] u8) or draw a rollout action into actions; rows whose
 * episode has ended get IDLE.  d == 0 starts the walk at the root; (e, d) == (0, 0) also zeroes skipped. */
int hwy_mcts_advance(const HwyMctsTree *t, int e, int d, const uint8_t *available, const double *reward,
                     const uint8_t *terminated, const uint8_t *truncated, void *stream);
/* End of episode e: add the last step's reward (f64 [n_roots]) to each walk that has not ended, back the return up
 * from the walk's node to the root and record leaf / returns [., e]. */
int hwy_mcts_backup(const HwyMctsTree *t, int e, const double *reward, void *stream);
/* recommended[r] = the root child with the largest count, ties by value then lowest action; decision += 1. */
int hwy_mcts_recommend(const HwyMctsTree *t, void *stream);
/* Subtree reuse: root r's child for actions[r] (int64) becomes the root, its subtree compacted to the front in index
 * order; roots with done[r] (u8) or without that child are cleared to a bare root.  actions = done = NULL clears every
 * tree. */
int hwy_mcts_reroot(const HwyMctsTree *t, const int64_t *actions, const uint8_t *done, void *stream);

/* ====================================================================== lane-keeping-v0
 * LaneKeepingEnv (envs/lane_keeping_env.py): one dynamical BicycleVehicle per env, no traffic, one thread per env.
 * lanes[0] is ("c", "d", 0), the StraightLane the episode starts on; lanes[1] is ("a", "b", 0), the SineLane queued
 * after it.  The ego spawns at (x0, y0) with heading0 and speed0, zero lateral speed and yaw rate.
 * attr[k] in 0 state, 1 derivative, 2 reference_state: the AttributesObservation columns in config order; each
 * observe draws 4 uniforms per noisy attribute (state, derivative) from the env's stream, in attribute order.
 * actions [n_envs][longitudinal + lateral] float32: (throttle, steering) of ContinuousAction in that order. */
#define HWY_LK_MAX_ATTR 3
typedef struct HwyLaneKeepingParams {
    int32_t frames;     /* simulation_frequency // policy_frequency (>= 1) */
    int32_t n_attr;     /* 1..HWY_LK_MAX_ATTR */
    int32_t attr[HWY_LK_MAX_ATTR];
    int32_t longitudinal, lateral, act_clip;
    int32_t max_episode_steps; /* TimeLimit: truncated once this many steps have run since the reset */
    int32_t autoreset;  /* HWY_AUTORESET_DISABLED or HWY_AUTORESET_SAME_STEP */
    double dt;          /* 1 / simulation_frequency */
    double state_noise, derivative_noise;
    double acc_lo, acc_hi, steer_lo, steer_hi;
    double x0, y0, heading0, speed0;
    HwyNetLane lanes[2];
} HwyLaneKeepingParams;
typedef struct HwyLaneKeepingState {
    int32_t n_envs, _pad;
    double *state;       /* DEVICE [6][n_envs]: x, y, heading, speed, lateral_speed, yaw_rate */
    int32_t *lane_phase; /* DEVICE [n_envs]: 0 on lanes[0] with lanes[1] queued, 1 on lanes[1] */
    int32_t *elapsed;    /* DEVICE [n_envs]: steps since the last reset */
    uint64_t *rng;       /* DEVICE [5][n_envs] */
} HwyLaneKeepingState;
/* Reset the envs with mask_a[e] || mask_b[e] (both NULL: every env): the scene of LaneKeepingEnv._reset, then the three
 * observes of AbstractEnv.reset (two inside define_spaces, whose values are discarded); obs [n_envs][n_attr][4] f64
 * takes the last one. */
int hwy_lane_keeping_reset(const HwyLaneKeepingParams *p, const HwyLaneKeepingState *s, const uint8_t *mask_a,
                           const uint8_t *mask_b, double *obs, void *stream);
/* One LaneKeepingEnv.step of every env: lane switch, act, observe (of the state before the step), `frames` RK4 frames,
 * reward 1 - (lat / width)^2 on the env's current lane; terminated = 0, truncated = elapsed >= max_episode_steps.
 * With autoreset = HWY_AUTORESET_SAME_STEP a truncated env writes its observation to final_obs, is reset as above and
 * obs takes the reset observation; final_obs rows of the other envs are left as they were. */
int hwy_lane_keeping_step(const HwyLaneKeepingParams *p, const HwyLaneKeepingState *s, const float *actions,
                          double *obs, double *final_obs, double *reward, uint8_t *terminated, uint8_t *truncated,
                          void *stream);

/* Kernel launches issued by the calling thread through this library since load (the
 * `gpu_launches` claim of bench.py). */
uint64_t hwy_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
