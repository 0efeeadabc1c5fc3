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

#define HWY_ABI_VERSION 13
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
    int32_t _pad_obs;
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

/* AbstractEnv.reset()'s _reset() for the envs whose mask byte is non-zero (mask == NULL:
 * all): HighwayEnv._create_road/_create_vehicles (highway_env.py:55-98,177-182) with
 * Vehicle.create_random (kinematics.py:50-104), drawing from each env's PCG64 stream in
 * the reference's order.  If obs != NULL also writes the reset observation
 * [n_envs][obs_vehicles_count][n columns] float32 of those envs. */
int hwy_highway_reset(const HwyHighwayParams *p, const HwyHighwayState *s, const uint8_t *mask,
                      float *obs, void *stream);

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
int hwy_highway_step(const HwyHighwayParams *p, const HwyHighwayState *s, const int32_t *action_i,
                     const float *action_f, float *obs, double *reward, uint8_t *terminated,
                     uint8_t *truncated, double *info_speed, uint8_t *info_crashed, int autoreset,
                     float *final_obs, void *stream);

/* The operator seam `_simulate` uses (envs/common/abstract.py:304-307 without action_type.act):
 * `n_substeps` times  Road.act()  (road/road.py:464-467)  then  Road.step(1 / simulation_frequency)  (:469-481)
 * on the stored state, and nothing else — no observation, reward, clock or reset.  The controlled vehicle acts like
 * ControlledVehicle.act(None) (its current target lane / speed); a ContinuousAction ego keeps the action dict given in
 * `action_f` ([n_envs, 2] in [-1, 1], as for hwy_highway_step) or the default {steering 0, acceleration 0} if NULL.
 * What BASELINE.md's "Road.act() + Road.step(dt)" timing runs. */
int hwy_highway_substeps(const HwyHighwayParams *p, const HwyHighwayState *s, int n_substeps, const float *action_f,
                         void *stream);

/* The SameStep autoreset half of hwy_highway_step on its own: re-spawn the envs whose
 * terminated | truncated byte is set and overwrite their rows of `obs` with the reset
 * observation (lets a caller time / schedule the two halves separately). */
int hwy_highway_autoreset(const HwyHighwayParams *p, const HwyHighwayState *s,
                          const uint8_t *terminated, const uint8_t *truncated, float *obs,
                          void *stream);


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
    int32_t merge_lane;         /* table index of ("b", "c", 2): slow ControlledVehicles there are penalised */
    int32_t _pad_merge;
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

/* IntersectionEnv._spawn_vehicle constants (envs/intersection_env.py:325-352). */
typedef struct HwyIntersectionSpawn {
    int32_t spawn_lane[4];      /* table index of ("o"+k, "ir"+k, 0) */
    double spawn_probability;   /* config["spawn_probability"] */
    const int32_t *route_table; /* DEVICE [n_lanes][4][HWY_NET_MAX_ROUTE]: plan_route_to(lane, "o"+k) */
    const int32_t *route_len;   /* DEVICE [n_lanes][4] */
    /* _make_vehicles (:245-323), used by hwy_intersection_reset */
    int32_t ego_lane;              /* table index of ("o0", "ir0", 0) */
    int32_t ego_destination;       /* k of config["destination"] == "o"+k; -1 (None): "o" + integers(1, 4) */
    int32_t initial_vehicle_count; /* config["initial_vehicle_count"] */
    int32_t _pad;
    int32_t *scratch;              /* DEVICE [2 * (n_envs + 1)] int32: work lists (envs being reset; the
                                    * step's 16-slot / 32-slot populations).  NULL: hwy_intersection_step
                                    * runs every env on 32 slots and hwy_intersection_reset is unavailable */
} HwyIntersectionSpawn;

/* observation size in floats PER ENV: Kinematics K*F, TimeToCollision 3*3*(horizon*policy_frequency),
 * OccupancyGrid 4*11*11; times n_agents when several vehicles are controlled */
int hwy_network_obs_size(const HwyNetParams *p);

/* AbstractEnv.step (abstract.py:259-285) on a general network: action [n_envs] int32
 * (DiscreteMetaAction labels, action.py:204).  graph is a DEVICE pointer. */
int hwy_network_step(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetState *s,
                     const int32_t *action, float *obs, double *reward, uint8_t *terminated,
                     uint8_t *truncated, double *info_speed, uint8_t *info_crashed, void *stream);

/* Same for intersection-v0 (s->vp == HWY_NET_GROUP_LARGE): RegulatedRoad rules every
 * int(simulation_frequency / 2) substeps, and after the observation the step's _clear_vehicles and
 * _spawn_vehicle(spawn_probability) drawing from s->rng (IntersectionEnv.step, :136-140). */
int hwy_intersection_step(const HwyNetParams *p, const HwyNetGraph *graph, const HwyIntersectionSpawn *spawn,
                          const HwyNetState *s, const int32_t *action, float *obs, double *reward,
                          uint8_t *terminated, uint8_t *truncated, double *info_speed,
                          uint8_t *info_crashed, void *stream);

/* The same with config["controlled_vehicles"] = p->n_agents > 1 (intersection-multi-agent-v0,
 * envs/intersection_env.py:376-420): action [n_envs][n_agents], obs [n_envs][n_agents][K][F]; reward is the mean
 * of the agents' rewards, terminated = any crashed or all arrived (:62-134); agents_reward / agents_terminated
 * [n_envs][n_agents] (optional) are _info's per-agent entries, which MultiAgentWrapper (abstract.py:468-477)
 * returns in place of the scalar reward / terminated. */
int hwy_intersection_step_agents(const HwyNetParams *p, const HwyNetGraph *graph, const HwyIntersectionSpawn *spawn,
                                 const HwyNetState *s, const int32_t *action, float *obs, double *reward,
                                 uint8_t *terminated, uint8_t *truncated, double *info_speed,
                                 uint8_t *info_crashed, double *agents_reward, uint8_t *agents_terminated,
                                 void *stream);

/* IntersectionEnv._reset / _make_vehicles (envs/intersection_env.py:119-122,245-323) on the device for the
 * envs with mask_a[e] | mask_b[e] (both NULL: every env): n-1 _spawn_vehicle draws, 3 s of warm-up simulation,
 * the challenger, the controlled vehicle (MDPVehicle on ("o0","ir0",0) at 60 + 5*normal(1)), the 20 m pruning;
 * all draws come from s->rng in the reference's order.  With final_obs, obs is first copied there (the
 * SameStep autoreset's info["final_obs"]); the fresh observation of the reset envs is written to obs. */
int hwy_intersection_reset(const HwyNetParams *p, const HwyNetGraph *graph, const HwyIntersectionSpawn *spawn,
                           const HwyNetState *s, const uint8_t *mask_a, const uint8_t *mask_b, float *obs,
                           float *final_obs, void *stream);

/* Test entries (the reference's own known-answer tests run against the device functions):
 * Road.neighbour_vehicles(v, lane) (road/road.py:483-547) for every vehicle v of every env — lane = query_lane
 * [n_envs*vp] or, when NULL, v's own lane — into front / rear [n_envs*vp] (slot index, -1 = None);
 * utils.rotated_rectangles_intersect (utils.py:115-125) for n pairs, rects [n][10] =
 * (cx, cy, length, width, angle) x 2 on the DEVICE. */
int hwy_debug_network_neighbours(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetState *s,
                                 const int32_t *query_lane, int32_t *front, int32_t *rear, void *stream);
int hwy_debug_rotated_rectangles_intersect(const double *rects, int n, int32_t *out, void *stream);

/* Road.act() + Road.step(dt) n_substeps times without an ego action, for the envs whose mask byte is
 * set (NULL: all): the 3 s warm-up of IntersectionEnv._make_vehicles (:271-278). */
int hwy_network_substeps(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetState *s,
                         const uint8_t *mask, int n_substeps, void *stream);

/* observation_type.observe() of the current state */
int hwy_network_observe(const HwyNetParams *p, const HwyNetGraph *graph, const HwyNetState *s,
                        float *obs, void *stream);

/* MergeEnv._make_vehicles + the Obstacle of _make_road (envs/merge_env.py:150-190) on the device: the MDPVehicle on
 * ("a","b",1) at s = 30, speed 30; three IDM vehicles on ("a","b", integers(2)) at position + uniform(-5, 5) with
 * speed + uniform(-1, 1); the merging vehicle on ("j","k",0) at s = 110, speed 20, target speed 30; and, in the
 * slot after the vehicles, the Obstacle (kind HWY_KIND_OBSTACLE) at the end of the ramp.  mask_a | mask_b select
 * the envs (both NULL: all); with obs, the fresh observation of those envs is written. */
typedef struct HwyMergeSpawn {
    int32_t lane_ab[2];      /* table indices of ("a","b",0), ("a","b",1) */
    int32_t lane_jk;         /* ("j","k",0) */
    int32_t ego_speed_index; /* MDPVehicle.speed_to_index(30) */
    double obstacle_x, obstacle_y;
} HwyMergeSpawn;
int hwy_merge_reset(const HwyNetParams *p, const HwyNetGraph *graph, const HwyMergeSpawn *spawn,
                    const HwyNetState *s, uint64_t *rng, const uint8_t *mask_a, const uint8_t *mask_b,
                    float *obs, void *stream);

/* UTurnEnv._make_vehicles (envs/u_turn_env.py:179-275) on the device: the MDPVehicle at the start of ("a","b",0),
 * speed 16, and six IDM vehicles made with make_on_lane(lane[v], longitudinal[v] + 2 normal(), speed[v] + 2 normal());
 * vehicle 1 also draws its DELTA (randomize_behavior); every vehicle gets plan_route_to("d") from a host-built
 * table indexed by the closest lane.  (The reference also sets ego.PURSUIT_TAU, an attribute nothing reads —
 * steering_control uses TAU_PURSUIT, vehicle/controller.py:28,159 — so there is nothing to restate.) */
typedef struct HwyUTurnSpawn {
    int32_t lane[8];             /* [0] ego lane ("a","b",0); [1..6] make_on_lane lanes */
    double longitudinal[8], speed[8];
    int32_t ego_speed_index, _pad;
    const int32_t *route_table;  /* DEVICE [n_lanes][HWY_NET_MAX_ROUTE]: plan_route_to("d") from each lane */
    const int32_t *route_len;    /* DEVICE [n_lanes] */
} HwyUTurnSpawn;
int hwy_u_turn_reset(const HwyNetParams *p, const HwyNetGraph *graph, const HwyUTurnSpawn *spawn,
                     const HwyNetState *s, uint64_t *rng, const uint8_t *mask_a, const uint8_t *mask_b,
                     float *obs, void *stream);

/* ExitEnv._create_vehicles (envs/exit_env.py:107-145) on the device: the MDPVehicle from Vehicle.create_random(speed=25,
 * lane ("0","1",0), spacing=ego_spacing); vehicles_count IDMVehicles on ("0","1", choice(lanes, p=lanes/sum)) at the
 * lane's speed limit, spacing 1 / vehicles_density, routed to "3", enable_lane_change=False.  State stride 32, s->count
 * is set to n_vehicles. */
typedef struct HwyExitSpawn {
    int32_t lanes_count, n_vehicles;   /* config["lanes_count"], 1 + config["vehicles_count"] */
    int32_t ego_speed_index, _pad;
    double ego_speed, ego_spacing, vehicles_density;
    double spawn_exp;                  /* np.exp(-5 / 40 * lanes_count) (vehicle/kinematics.py:95) */
    double cdf[HWY_MAX_LANES];         /* Generator.choice(p=lanes / lanes.sum()): p.cumsum() / cumsum[-1] */
    int32_t route_12, route_23;        /* encoded route entries ("1","2",None), ("2","3",None) */
} HwyExitSpawn;
int hwy_exit_reset(const HwyNetParams *p, const HwyNetGraph *graph, const HwyExitSpawn *spawn, const HwyNetState *s,
                   uint64_t *rng, const uint8_t *mask_a, const uint8_t *mask_b, float *obs, void *stream);

/* TwoWayEnv._make_vehicles (envs/two_way_env.py:113-158) on the device: the MDPVehicle on ("a","b",1) at s = 30,
 * three IDM vehicles ahead at 70 + 40 i + 10 normal() with speed 24 + 2 normal(), two oncoming ones on ("b","a",0)
 * at 200 + 100 i + 10 normal() with speed 20 + 5 normal(); all traffic has enable_lane_change=False. */
typedef struct HwyTwoWaySpawn {
    int32_t lane_ab1, lane_ba0; /* table indices of ("a","b",1) and ("b","a",0) */
    int32_t ego_speed_index, _pad;
} HwyTwoWaySpawn;
int hwy_two_way_reset(const HwyNetParams *p, const HwyNetGraph *graph, const HwyTwoWaySpawn *spawn,
                      const HwyNetState *s, uint64_t *rng, const uint8_t *mask_a, const uint8_t *mask_b,
                      float *obs, void *stream);

/* RoundaboutEnv._make_vehicles (envs/roundabout_env.py:317-391) on the device.  Per traffic
 * vehicle the env's numpy stream yields normal (longitudinal), normal (speed),
 * choice(destinations), uniform (DELTA); routes come from a host-built table of
 * ControlledVehicle.plan_route_to results (vehicle/controller.py:71-87). */
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

/* Re-spawn the envs selected by mask_a | mask_b (both NULL: all) from rng[5*n_envs] (layout as
 * HwyHighwayState.rng); if obs != NULL also write their reset observation. */
int hwy_roundabout_reset(const HwyNetParams *p, const HwyNetGraph *graph, const HwyRoundaboutSpawn *spawn,
                         const HwyNetState *s, uint64_t *rng, const uint8_t *mask_a, const uint8_t *mask_b,
                         float *obs, void *stream);

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

/* LidarObservation (observation.py:678-769): obs [n_envs][agents][cells][2] float32 (distance, relative radial speed) */
typedef struct HwyLidarParams {
    int32_t cells, normalize;
    double maximum_range;
} HwyLidarParams;
int hwy_observe_lidar(const HwyObsView *view, const HwyLidarParams *p, const uint8_t *mask_a, const uint8_t *mask_b,
                      float *obs, void *stream);

/* Kernel launches issued by the calling thread through this library since load (the
 * `gpu_launches` claim of bench.py). */
uint64_t hwy_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
