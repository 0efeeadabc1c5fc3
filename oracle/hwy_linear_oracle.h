/*
 * hwy_linear_oracle.h — CPU restatement of LinearVehicle / AggressiveVehicle / DefensiveVehicle traffic on the
 * straight highway family (vehicle/behavior.py:350-583).  TEST INFRASTRUCTURE ONLY, like hwy_oracle.h: nothing in the
 * product may include, link or call it.  The library is hwy_oracle.c plus hwy_linear_oracle.c; it uses hwy_oracle.h's
 * config, state and batch structs unchanged and keeps each vehicle's parameters in a separate buffer
 * params[V][5] = ACCELERATION_PARAMETERS (3), STEERING_PARAMETERS (2), zero for the controlled vehicle.  The config's
 * time_wanted and lane_change_min_acc_gain are the traffic class's (2.5; 0.2 Linear, 1.0 Aggressive / Defensive).
 * Parity is pinned by tests/test_linear_traffic_spec.py against the fixtures of oracle/gen_linear_golden.py.
 */
#ifndef HWY_LINEAR_ORACLE_H
#define HWY_LINEAR_ORACLE_H

#include "hwy_oracle.h"

#ifdef __cplusplus
extern "C" {
#endif

/* randomize_behavior's ranges (behavior.py:353-371, 406-415): lo = RANGE[0], span = RANGE[1] - RANGE[0] (numpy) */
typedef struct OrcLinearTraffic {
    double acc_lo[3], acc_span[3], steer_lo[2], steer_span[2];
} OrcLinearTraffic;

/* the two controllers on plain inputs (LinearVehicle.acceleration / steering_control, behavior.py:417-502) */
double orc_linear_acceleration(const double a[3], double target_speed, double speed, int has_front, double front_speed,
                               double d, double distance_wanted, double time_wanted);
double orc_linear_steering(const double p[2], double lane_heading, double heading, double lat, double speed);

void orc_linear_highway_reset(const OrcHighwayCfg *cfg, const OrcLinearTraffic *t, OrcPcg64 *rng,
                              OrcHighwayState *st, double *params);
void orc_linear_highway_step(const OrcHighwayCfg *cfg, const OrcLinearTraffic *t, OrcHighwayState *st,
                             const double *params, int action_i, const float *action_f, float *obs, double *reward,
                             int32_t *terminated, int32_t *truncated);
void orc_linear_highway_substeps(const OrcHighwayCfg *cfg, OrcHighwayState *st, const double *params, int substeps);

/* batched drivers as orc_highway_*_batch; params [n_envs][V][5] */
void orc_linear_highway_reset_batch(const OrcHighwayCfg *cfg, const OrcLinearTraffic *t, OrcBatch *b, double *params,
                                    const uint8_t *mask, float *obs, int threads);
void orc_linear_highway_step_batch(const OrcHighwayCfg *cfg, const OrcLinearTraffic *t, OrcBatch *b, double *params,
                                   const int32_t *action_i, const float *action_f, float *obs, double *reward,
                                   uint8_t *terminated, uint8_t *truncated, int autoreset, int threads);
void orc_linear_highway_substeps_batch(const OrcHighwayCfg *cfg, OrcBatch *b, double *params, int substeps,
                                       int threads);

#ifdef __cplusplus
}
#endif
#endif
