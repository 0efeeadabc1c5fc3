/*
 * hwy_linear_oracle.c — scalar CPU restatement of LinearVehicle / AggressiveVehicle / DefensiveVehicle traffic on
 * the straight highway family (vehicle/behavior.py:350-583).  TEST INFRASTRUCTURE ONLY — see hwy_linear_oracle.h.
 *
 * The IDM restatement of hwy_oracle.c is compiled into this library unchanged (it is #included below, so its static
 * helpers — lanes, neighbour search, collisions, controlled-vehicle and ContinuousAction acts, observation, reward —
 * are shared rather than copied).  What this file adds are the parts the traffic model changes: the traffic
 * vehicle's act (acceleration, MOBIL, steering), the reset draws, and step / substeps / batch drivers that call them.
 * Build as hwy_oracle.c: gcc -O2 -ffp-contract=off (explicit fma() where numpy fuses).
 */
#include "hwy_oracle.c"

#include "hwy_linear_oracle.h"

/* python min(x, 0) */
static inline double py_min0(double x) { return 0 < x ? 0.0 : x; }

/* vehicle/behavior.py:417-465 LinearVehicle.acceleration, given the ego's target speed (getattr(ego, "target_speed",
 * ego.speed)) and speed and, for a front vehicle (has_front), its speed and the lane distance d to it:
 * np.dot(ACCELERATION_PARAMETERS, [vt, dv, dp]); numpy's BLAS ddot on 3-vectors is fma(a2, b2, fma(a1, b1, a0 * b0)). */
double orc_linear_acceleration(const double a[3], double target_speed, double speed, int has_front, double front_speed,
                               double d, double distance_wanted, double time_wanted) {
    double vt = target_speed - speed, dv = 0, dp = 0;
    double d_safe = distance_wanted + fmax(speed, 0) * time_wanted;
    if (has_front) {
        dv = py_min0(front_speed - speed);
        dp = py_min0(d - d_safe);
    }
    return fma(a[2], dp, fma(a[1], dv, a[0] * vt));
}

/* vehicle/behavior.py:467-502 LinearVehicle.steering_control on a StraightLane (heading_at = the lane heading), given
 * the lateral coordinate on the target lane: np.dot(STEERING_PARAMETERS, features) = fma(p1, f1, p0 * f0).
 * not_zero(speed) ** 2 is a python float power, i.e. the libm pow, which is not always the correctly rounded x * x
 * (and which gcc would fold to x * x for a literal 2). */
double orc_linear_steering(const double p[2], double lane_heading, double heading, double lat, double speed) {
    static volatile double two = 2.0;
    double nz = orc_not_zero(speed);
    double f0 = orc_wrap_to_pi(lane_heading - heading) * VEH_LENGTH / nz;
    double f1 = -lat * VEH_LENGTH / pow(nz, two);
    return fma(p[1], f1, p[0] * f0);
}

/* acceleration(ego_vehicle=ego, front_vehicle=front) with the CALLER's parameters a[3]; ego < 0 (None) gives 0 */
static double linear_acceleration(const World *w, const double *a, int ego, int front) {
    const OrcHighwayCfg *c = w->c;
    const OrcHighwayState *s = w->s;
    if (ego < 0) return 0;
    double ts = s->kind[ego] == ORC_KIND_VEHICLE ? s->speed[ego] : s->target_speed[ego];
    double d = front >= 0 ? lane_distance_to(w, ego, front) : 0;
    return orc_linear_acceleration(a, ts, s->speed[ego], front >= 0, front >= 0 ? s->speed[front] : 0, d,
                                   c->distance_wanted, c->time_wanted);
}

/* vehicle/behavior.py:265-324 mobil with LinearVehicle.acceleration (the caller's parameters for every vehicle) */
static int linear_mobil(const World *w, const double *a, int v, int lane_index) {
    const OrcHighwayCfg *c = w->c;
    int new_preceding, new_following;
    neighbour_vehicles(w, v, lane_index, &new_preceding, &new_following);
    double new_following_a = linear_acceleration(w, a, new_following, new_preceding);
    double new_following_pred_a = linear_acceleration(w, a, new_following, v);
    if (new_following_pred_a < -c->lane_change_max_braking_imposed) return 0;
    int old_preceding, old_following;
    neighbour_vehicles(w, v, w->s->lane[v], &old_preceding, &old_following);
    double self_pred_a = linear_acceleration(w, a, v, new_preceding);
    double self_a = linear_acceleration(w, a, v, old_preceding);
    double old_following_a = linear_acceleration(w, a, old_following, v);
    double old_following_pred_a = linear_acceleration(w, a, old_following, old_preceding);
    double jerk = self_pred_a - self_a +
                  c->politeness * (new_following_pred_a - new_following_a + old_following_pred_a -
                                   old_following_a);
    if (jerk < c->lane_change_min_acc_gain) return 0;
    return 1;
}

/* vehicle/behavior.py:219-263 change_lane_policy (desired_gap with the class's TIME_WANTED = cfg time_wanted) */
static void linear_change_lane_policy(World *w, const double *a, int v) {
    const OrcHighwayCfg *c = w->c;
    OrcHighwayState *s = w->s;
    if (s->lane[v] != s->target_lane[v]) {
        for (int o = 0; o < w->V; o++) {
            if (o != v && s->lane[o] != s->target_lane[v] && s->kind[o] != ORC_KIND_VEHICLE &&
                s->target_lane[o] == s->target_lane[v]) {
                double d = lane_distance_to(w, v, o);
                double d_star = desired_gap(w, v, o);
                if (0 < d && d < d_star) {
                    s->target_lane[v] = s->lane[v];
                    break;
                }
            }
        }
        return;
    }
    if (!(c->lane_change_delay < s->timer[v])) return; /* utils.do_every, utils.py:27-28 */
    s->timer[v] = 0;
    int cand[2], nc = 0;
    if (s->lane[v] > 0) cand[nc++] = s->lane[v] - 1;
    if (s->lane[v] < c->lanes_count - 1) cand[nc++] = s->lane[v] + 1;
    for (int k = 0; k < nc; k++) {
        if (!lane_reachable(&w->lanes[cand[k]], s->x[v], s->y[v])) continue;
        if (fabs(s->speed[v]) < 1) continue;
        if (linear_mobil(w, a, v, cand[k])) s->target_lane[v] = cand[k];
    }
}

/* IDMVehicle.act (behavior.py:93-137) with LinearVehicle's acceleration and steering_control; collect_data (:389-392,
 * regression features appended to vehicle.data) has no effect on the dynamics and is not restated */
static void linear_act(World *w, const double *params, int v) {
    const OrcHighwayCfg *c = w->c;
    OrcHighwayState *s = w->s;
    if (s->crashed[v]) return;
    const double *a = params + 5 * v;
    follow_road(w, v);
    linear_change_lane_policy(w, a, v);
    const Lane *L = &w->lanes[s->target_lane[v]];
    double lc_s, lc_lat;
    lane_local(L, s->x[v], s->y[v], &lc_s, &lc_lat);
    double steering = orc_linear_steering(a + 3, L->heading, s->heading[v], lc_lat, s->speed[v]);
    steering = clipd(steering, -MAX_STEERING_ANGLE, MAX_STEERING_ANGLE);
    int front, rear;
    neighbour_vehicles(w, v, s->lane[v], &front, &rear);
    double acc = linear_acceleration(w, a, v, front);
    if (s->lane[v] != s->target_lane[v]) {
        neighbour_vehicles(w, v, s->target_lane[v], &front, &rear);
        double tacc = linear_acceleration(w, a, v, front);
        acc = fmin(acc, tacc);
    }
    acc = clipd(acc, -c->acc_max, c->acc_max);
    w->act_steer[v] = steering;
    w->act_accel[v] = acc;
}

/* road/road.py:464-467 Road.act with linear traffic */
static void linear_road_act(World *w, const double *params) {
    for (int v = 0; v < w->V; v++) {
        switch (w->s->kind[v]) {
        case ORC_KIND_IDM: linear_act(w, params, v); break;
        case ORC_KIND_MDP: controlled_act(w, v, -1); break;
        default: break;
        }
    }
}

void orc_linear_highway_step(const OrcHighwayCfg *c, const OrcLinearTraffic *t, OrcHighwayState *s,
                             const double *params, int action_i, const float *action_f, float *obs, double *reward,
                             int32_t *terminated, int32_t *truncated) {
    (void)t;
    World w;
    double *act_buf = (double *)malloc(sizeof(double) * 2 * c->n_vehicles);
    world_init(&w, c, s, act_buf);
    int frames = c->simulation_frequency / c->policy_frequency;
    double dt = 1.0 / c->simulation_frequency;
    s->time[0] += 1.0 / c->policy_frequency;
    for (int frame = 0; frame < frames; frame++) {
        if (frame == 0) {
            if (c->action_type == 0)
                mdp_act(&w, 0, action_i);
            else
                continuous_act(&w, 0, action_f);
        }
        linear_road_act(&w, params);
        road_step(&w, dt);
    }
    if (obs) orc_highway_observe(c, s, obs);
    reward_done(&w, reward, terminated, truncated);
    free(act_buf);
}

void orc_linear_highway_substeps(const OrcHighwayCfg *c, OrcHighwayState *s, const double *params, int substeps) {
    World w;
    double *act_buf = (double *)malloc(sizeof(double) * 2 * c->n_vehicles);
    world_init(&w, c, s, act_buf);
    double dt = 1.0 / c->simulation_frequency;
    for (int k = 0; k < substeps; k++) {
        linear_road_act(&w, params);
        road_step(&w, dt);
    }
    free(act_buf);
}

/* orc_highway_reset with LinearVehicle.randomize_behavior (behavior.py:406-415): uniform(size=3), uniform(size=2)
 * mapped by RANGE[0] + u * (RANGE[1] - RANGE[0]), before the inherited DELTA draw; the ego's row of params is zero */
void orc_linear_highway_reset(const OrcHighwayCfg *c, const OrcLinearTraffic *t, OrcPcg64 *rng, OrcHighwayState *s,
                              double *params) {
    Lane lanes[ORC_MAX_LANES];
    make_lanes(c, lanes);
    int V = c->n_vehicles;
    s->time[0] = 0;
    for (int v = 0; v < V; v++) {
        int is_ego = v == 0;
        int id;
        if (is_ego && c->initial_lane_id >= 0)
            id = c->initial_lane_id;
        else
            id = (int)orc_rng_choice(rng, c->lanes_count);
        const Lane *L = &lanes[id];
        double speed;
        if (is_ego)
            speed = c->ego_speed;
        else
            speed = orc_rng_uniform(rng, 0.7 * L->speed_limit, 0.8 * L->speed_limit);
        double spacing = is_ego ? c->ego_spacing : 1 / c->vehicles_density;
        double default_spacing = 12 + 1.0 * speed;
        double offset = spacing * default_spacing * c->spawn_exp;
        double x0;
        if (v > 0) {
            x0 = lane_s(L, s->x[0], s->y[0]);
            for (int j = 1; j < v; j++) x0 = fmax(x0, lane_s(L, s->x[j], s->y[j]));
        } else {
            x0 = 3 * offset;
        }
        x0 += offset * orc_rng_uniform(rng, 0.9, 1.1);
        lane_position(L, x0, 0, &s->x[v], &s->y[v]);
        s->heading[v] = L->heading;
        s->speed[v] = speed;
        s->lane[v] = closest_lane(lanes, c->lanes_count, s->x[v], s->y[v], s->heading[v]);
        s->target_lane[v] = s->lane[v];
        s->target_speed[v] = speed;
        s->crashed[v] = 0;
        s->has_impact[v] = 0;
        s->impact_x[v] = s->impact_y[v] = 0;
        s->timer[v] = 0;
        s->delta[v] = 4.0;
        double *p = params + 5 * v;
        memset(p, 0, 5 * sizeof(double));
        if (is_ego) {
            s->check_collisions[v] = 1;
            if (c->action_type == 0) {
                s->kind[v] = ORC_KIND_MDP;
                s->speed_index[0] = speed_to_index(c, s->target_speed[v]);
                s->target_speed[v] = c->target_speeds[s->speed_index[0]];
            } else {
                s->kind[v] = ORC_KIND_VEHICLE;
                s->speed_index[0] = -1;
            }
        } else {
            s->kind[v] = ORC_KIND_IDM;
            s->check_collisions[v] = c->others_check_collisions;
            s->timer[v] = py_mod((s->x[v] + s->y[v]) * M_PI, c->lane_change_delay);
            for (int k = 0; k < 3; k++) p[k] = t->acc_lo[k] + orc_rng_uniform(rng, 0.0, 1.0) * t->acc_span[k];
            for (int k = 0; k < 2; k++) p[3 + k] = t->steer_lo[k] + orc_rng_uniform(rng, 0.0, 1.0) * t->steer_span[k];
            s->delta[v] = orc_rng_uniform(rng, c->delta_lo, c->delta_hi);
        }
    }
}

/* ------------------------------------------------------------------ batched driver */

typedef struct {
    const OrcHighwayCfg *c;
    const OrcLinearTraffic *t;
    OrcBatch *b;
    double *params; /* [n_envs][V][5] */
    const uint8_t *mask;
    const int32_t *action_i;
    const float *action_f;
    float *obs;
    double *reward;
    uint8_t *terminated, *truncated;
    int autoreset, e0, e1, mode;
} LinJob;

static void *linear_job_run(void *arg) {
    LinJob *j = (LinJob *)arg;
    const OrcHighwayCfg *c = j->c;
    size_t obs_sz = (size_t)c->obs_vehicles_count * orc_highway_obs_columns(c);
    for (int e = j->e0; e < j->e1; e++) {
        OrcHighwayState s;
        bind_env(c, j->b, e, &s);
        double *params = j->params + (size_t)e * c->n_vehicles * 5;
        if (j->mode == 0) {
            if (j->mask && !j->mask[e]) continue;
            orc_linear_highway_reset(c, j->t, &j->b->rng[e], &s, params);
            if (j->obs) orc_highway_observe(c, &s, j->obs + obs_sz * e);
        } else if (j->mode == 1) {
            double r;
            int32_t te, tr;
            orc_linear_highway_step(c, j->t, &s, params, j->action_i ? j->action_i[e] : 0,
                                    j->action_f ? j->action_f + 2 * (size_t)e : NULL,
                                    j->obs ? j->obs + obs_sz * e : NULL, &r, &te, &tr);
            j->reward[e] = r;
            j->terminated[e] = (uint8_t)te;
            j->truncated[e] = (uint8_t)tr;
            if (j->autoreset && (te || tr)) {
                orc_linear_highway_reset(c, j->t, &j->b->rng[e], &s, params);
                if (j->obs) orc_highway_observe(c, &s, j->obs + obs_sz * e);
            }
        } else {
            orc_linear_highway_substeps(c, &s, params, j->autoreset);
        }
    }
    return NULL;
}

static void linear_run_jobs(LinJob *proto, int n_envs, int threads) {
    if (threads < 1) threads = 1;
    if (threads > n_envs) threads = n_envs > 0 ? n_envs : 1;
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * threads);
    LinJob *jobs = (LinJob *)malloc(sizeof(LinJob) * threads);
    for (int k = 0; k < threads; k++) {
        jobs[k] = *proto;
        jobs[k].e0 = (int)((long long)n_envs * k / threads);
        jobs[k].e1 = (int)((long long)n_envs * (k + 1) / threads);
        if (threads == 1)
            linear_job_run(&jobs[k]);
        else
            pthread_create(&th[k], NULL, linear_job_run, &jobs[k]);
    }
    if (threads > 1)
        for (int k = 0; k < threads; k++) pthread_join(th[k], NULL);
    free(th);
    free(jobs);
}

void orc_linear_highway_reset_batch(const OrcHighwayCfg *c, const OrcLinearTraffic *t, OrcBatch *b, double *params,
                                    const uint8_t *mask, float *obs, int threads) {
    LinJob j;
    memset(&j, 0, sizeof(j));
    j.c = c;
    j.t = t;
    j.b = b;
    j.params = params;
    j.mask = mask;
    j.obs = obs;
    j.mode = 0;
    linear_run_jobs(&j, b->n_envs, threads);
}

void orc_linear_highway_step_batch(const OrcHighwayCfg *c, const OrcLinearTraffic *t, OrcBatch *b, double *params,
                                   const int32_t *action_i, const float *action_f, float *obs, double *reward,
                                   uint8_t *terminated, uint8_t *truncated, int autoreset, int threads) {
    LinJob j;
    memset(&j, 0, sizeof(j));
    j.c = c;
    j.t = t;
    j.b = b;
    j.params = params;
    j.action_i = action_i;
    j.action_f = action_f;
    j.obs = obs;
    j.reward = reward;
    j.terminated = terminated;
    j.truncated = truncated;
    j.autoreset = autoreset;
    j.mode = 1;
    linear_run_jobs(&j, b->n_envs, threads);
}

void orc_linear_highway_substeps_batch(const OrcHighwayCfg *c, OrcBatch *b, double *params, int substeps,
                                       int threads) {
    LinJob j;
    memset(&j, 0, sizeof(j));
    j.c = c;
    j.b = b;
    j.params = params;
    j.autoreset = substeps;
    j.mode = 2;
    linear_run_jobs(&j, b->n_envs, threads);
}
