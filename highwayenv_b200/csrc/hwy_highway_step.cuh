// hwy_highway_step.cuh — the body of the highway step kernels, included by highway_step_kernel (LINEAR = false),
// highway_linear_step_kernel (LINEAR = true) and highway_multi_step_kernel (MULTI = true: several controlled
// vehicles) in hwy_highway.cu.  In scope: TPE, AL, LINEAR, MULTI, the kernel parameters and
// `const HwyLinearTraffic* T`.  See the comment above highway_step_kernel.
    constexpr int NW = TPE / 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    EnvShared<TPE>* smem = reinterpret_cast<EnvShared<TPE>*>(smem_raw);
    const int V = P.n_vehicles;
    // DENSE: env `sub` of the block owns the V threads from sub * V; the threads past EPB * V own no vehicle (i = V,
    // active = false): they keep the last env's shared-memory address but neither load nor store.  Otherwise env
    // `sub` owns the TPE threads from sub * TPE.
    const int EPB = DENSE ? dense_epb : blockDim.x / TPE;
    const int seg = threadIdx.x / (DENSE ? V : TPE);
    const int sub = DENSE && seg >= EPB ? EPB - 1 : seg;
    const int i = DENSE ? (seg < EPB ? threadIdx.x - seg * V : V) : threadIdx.x % TPE;
    const bool active = i < V;
    const int env = blockIdx.x * EPB + sub;
    const bool env_ok = (!DENSE || active) && env < S.n_envs;  // surplus envs of the last block mirror the last env
    const int e = env < S.n_envs ? env : S.n_envs - 1;
    EnvShared<TPE>& sm = smem[sub];
    LinearShared<TPE>* lsm = nullptr;
    if constexpr (LINEAR) lsm = reinterpret_cast<LinearShared<TPE>*>(smem + EPB) + sub;
    MultiShared<TPE>* msm = nullptr;
    if constexpr (MULTI) msm = reinterpret_cast<MultiShared<TPE>*>(smem + EPB) + sub;
    const size_t slot = (size_t)e * S.vp + (active ? i : 0);
    const bool aligned = AL || lanes_aligned(P);
    const bool congruent = AL || lanes_congruent(P);

    VehicleRegs r;
    if constexpr (DENSE) {
        r = {};
        if (active) load_vehicle(S, slot, r);
    } else {
        load_vehicle(S, slot, r);
    }
    const int kind = meta_kind(r.meta);
    int speed_index = (!MULTI && i == 0) ? S.speed_index[e] : 0;  // MULTI: read on frame 0, per controlled vehicle
    // MULTI: this slot is a controlled vehicle (MDPVehicle or Vehicle), the agent-th one of its env
    const bool controlled = MULTI && active && (kind == HWY_KIND_MDP || kind == HWY_KIND_VEHICLE);
    int agent = 0;
    double act_steer = 0.0, act_accel = 0.0;
    // autoreset < 0 (hwy_highway_substeps): -autoreset times Road.act() + Road.step(dt) and nothing else — no
    // action_type.act, no observation / reward / clock; the controlled vehicle acts like ControlledVehicle.act(None)
    const int substeps_only = autoreset < 0 ? -autoreset : 0;
    const int frames = substeps_only ? substeps_only : P.simulation_frequency / P.policy_frequency;
    const double dt = 1.0 / P.simulation_frequency;

    // ---- static masks
    {
        uint32_t b_cc = __ballot_sync(0xffffffffu, active && (r.meta & HWY_META_CHECK_COLLISIONS));
        uint32_t b_ctrl = __ballot_sync(0xffffffffu, active && kind != HWY_KIND_VEHICLE);
        uint32_t b_ego = 0;
        if constexpr (MULTI) b_ego = __ballot_sync(0xffffffffu, controlled);
        if constexpr (DENSE) {
            if (i < NW) sm.cc[i] = sm.ctrl[i] = sm.mid[i] = 0;
            if constexpr (MULTI)
                if (i < NW) msm->ego[i] = 0;
            if (active) {
                sm.last_will[i] = -1;
                sm.crash_hit[i] = 0;
            }
        } else {
            if ((i & 31) == 0) {
                sm.cc[i >> 5] = b_cc;
                sm.ctrl[i >> 5] = b_ctrl;
                sm.mid[i >> 5] = 0;
                if constexpr (MULTI) msm->ego[i >> 5] = b_ego;
            }
            sm.last_will[i] = -1;
            sm.crash_hit[i] = 0;
        }
        if (i < NW) sm.ok_left[i] = sm.ok_right[i] = 0;
        if (i == 0) sm.n_items = 0;
        if (active) sm.delta[i] = r.delta;
        if constexpr (LINEAR) {
            if (active) {
                const double* lp = T->params + slot * HWY_LINEAR_PARAMS;
                for (int k = 0; k < 3; ++k) lsm->acc[k][i] = lp[k];
                for (int k = 0; k < 2; ++k) lsm->steer[k][i] = lp[3 + k];
            }
        }
        if constexpr (DENSE) {
            __syncthreads();  // (once per launch) the zeroed words before the env segments OR their bits in
            segment_or(sm.cc, b_cc, i, V);
            segment_or(sm.ctrl, b_ctrl, i, V);
            if constexpr (MULTI) segment_or(msm->ego, b_ego, i, V);
        }
    }
    const IdmK K = make_idm(P);
    // all-pairs gate (every vehicle checks collisions): rank-pruned sweep; a single checking vehicle (highway-fast)
    // already costs one pre-check per thread
    const bool pruned = P.others_check_collisions != 0;
    int p = 1;
    // frame 0 takes its ranks from the order the last launch stored, once build_frame has checked it (sm.f[1] is the
    // previous frame of frame 0; the barrier after frame 0's publish orders these stores)
    if (active) stage_stored_order(sm.f[1], i, V, r.meta);
    PHASE_INIT();
    PHASE_MARK(0);  // load + static masks

    // One iteration = stage the current state, derive its masks (+ the collision sweep of the
    // substep that produced it), then — except after the last substep — act and integrate.
    for (int frame = 0;; ++frame) {
        p ^= 1;
        Frame<TPE>& F = sm.f[p];
        const bool acts = frame < frames;  // the last frame only feeds the collision sweep and the epilogue
        publish<TPE, LINEAR, DENSE>(P, F, i, active, r, kWarpOrder<TPE, DENSE> && acts);
        if (DENSE && active && acts) clear_masks(F, i, V);
        PHASE_MARK(1);  // publish
        env_sync<TPE>();
        PHASE_MARK(2);  // barrier after publish
        if (i < NW) sm.mid[i] = sm.ok_left[i] = sm.ok_right[i] = 0;  // all readers are past phase B
        if (i == 0) sm.n_items = 0;
        // warp w finds the road order of env w (a dense block has more warps than envs: V > 32)
        if constexpr (kWarpOrder<TPE, DENSE>)
            if ((int)(threadIdx.x >> 5) < EPB)
                warp_order(smem[threadIdx.x >> 5].f[p], smem[threadIdx.x >> 5].f[p ^ 1], V, acts ? P.lanes_count : 0);
        // frame 0: masks only — the sweep of the stored state ran at the end of the substep that
        // produced it (previous launch).  Later: Road.step's sweep (road/road.py:477-481).  The last frame: ranks and
        // the sweep, no masks.
        const bool single =
            build_frame<TPE, DENSE>(P, sm, F, i, active, aligned, r, dt, frame > 0, acts, pruned, sm.f[p ^ 1]);
        PHASE_MARK(3);  // ranks, masks, sweep pass 1
        if (pruned && frame > 0) {  // uniform over the grid
            env_sync_phase<TPE, 3>();
            sweep_pruned(sm, F, V, i, active, dt);
        }
        env_sync_phase<TPE, 3>();
        PHASE_MARK(4);  // barrier after build
        if (active && frame > 0 && (!single || i == 0)) apply_collisions(sm, F, i, r, dt, single);
        PHASE_MARK(5);  // sweep pass 2
        if (frame == frames) break;

        // ---- action_type.act(action) on the first frame (abstract.py:294-304)
        if (frame == 0) {
            if constexpr (MULTI) {  // (the ego mask is complete: two barriers since the static masks)
                for (int w = 0; w < NW; ++w)
                    agent += __popc(w < (i >> 5) ? msm->ego[w] : (w == (i >> 5) ? msm->ego[w] & ((1u << (i & 31)) - 1u) : 0u));
                if (controlled && agent < P.n_agents) speed_index = S.speed_index[(size_t)e * P.n_agents + agent];
            }
            // MULTI: MultiAgentAction hands action k to controlled vehicle k (action.py:301-333); a plain action type
            // acts on the first one only, the others act(None) (abstract.py:294-304, Road.act)
            // (a controlled slot past the n_agents-th, which only a hand-made state has, acts(None) and keeps no index)
            const bool own_action = MULTI && agent < P.n_agents && (P.multi_action || agent == 0);
            const size_t act_row = MULTI && P.multi_action ? (size_t)e * P.n_agents + agent : (size_t)e;
            if (MULTI ? controlled : i == 0) {
                if (kind == HWY_KIND_MDP) {
                    // MDPVehicle.act (controller.py:295-315) + ControlledVehicle.act lane part
                    // (:99-124); labels action.py:204.  follow_road (:135-143) cannot change the
                    // target on the single-road highway graph (next_lane hits KeyError,
                    // road/road.py:129-130).
                    int a;
                    if constexpr (MULTI)
                        a = (substeps_only || !own_action) ? 1 : action_i[act_row];
                    else
                        a = substeps_only ? 1 : action_i[e];  // substeps only: act(None) = IDLE
                    if (a == 3 || a == 4) {
                        int idx = speed_to_index(P, r.speed) + (a == 3 ? 1 : -1);
                        idx = max(0, min(idx, P.n_target_speeds - 1));
                        speed_index = idx;
                        r.target_speed = P.target_speeds[idx];
                        F.ts[MULTI ? i : 0] = r.target_speed;
                    } else if (a == 0 || a == 2) {
                        int old = meta_target(r.meta);
                        int id = old + (a == 2 ? 1 : -1);
                        id = max(0, min(id, P.lanes_count - 1));
                        if (lane_reachable(P.lanes[id], r.x, r.y)) {
                            r.meta = meta_set_target(r.meta, id);
                            if constexpr (MULTI) {  // (several controlled vehicles may share a mask word)
                                F.tgt[i] = (unsigned char)id;
                                atomicAnd(&F.tm[old][i >> 5], ~(1u << (i & 31)));
                                atomicOr(&F.tm[id][i >> 5], 1u << (i & 31));
                            } else {
                                F.tgt[0] = (unsigned char)id;
                                F.tm[old][0] &= ~1u;
                                F.tm[id][0] |= 1u;
                            }
                        }
                    }
                } else {
                    // ContinuousAction.get_action/act (action.py:136-162): Box is float32 and
                    // lmap (utils.py:31-33) stays in float32 (NEP 50 weak python scalars)
                    // (substeps only: the vehicle's current action dict, or the default {0, 0} when none is given —
                    // lmap(0) of the symmetric default ranges)
                    const size_t row = MULTI ? act_row : (size_t)e;
                    float a0 = action_f ? action_f[2 * row] : 0.0f, a1 = action_f ? action_f[2 * row + 1] : 0.0f;
                    if (P.act_clip) {
                        a0 = fminf(fmaxf(a0, -1.0f), 1.0f);
                        a1 = fminf(fmaxf(a1, -1.0f), 1.0f);
                    }
                    float acc = __fadd_rn((float)P.acc_lo,
                                          __fdiv_rn(__fmul_rn(__fsub_rn(a0, -1.0f),
                                                              (float)(P.acc_hi - P.acc_lo)), 2.0f));
                    float st = __fadd_rn((float)P.steer_lo,
                                         __fdiv_rn(__fmul_rn(__fsub_rn(a1, -1.0f),
                                                             (float)(P.steer_hi - P.steer_lo)), 2.0f));
                    act_accel = (double)acc;
                    act_steer = (double)st;
                    if (MULTI && !own_action) {  // Vehicle.act(None) keeps the action dict it was created with
                        act_accel = 0.0;
                        act_steer = 0.0;
                    }
                }
            }
            env_sync<TPE>();
        }

        PHASE_MARK(6);  // ego action (+ barrier on frame 0)
        // ---- Road.act() (road/road.py:464-467), phase A1: own-lane IDM; lane-change policy set-up
        const int lane = meta_lane(r.meta);
        const int tgt0 = meta_target(r.meta);
        const bool crashed = (r.meta & HWY_META_CRASHED) != 0;
        const bool idm_active = active && kind == HWY_KIND_IDM && !crashed;  // behavior.py:102-103
        bool is_mid = false, fired = false;
        double acc = 0.0, free_i = 0.0;
        if (idm_active) {
            if constexpr (!LINEAR)
                free_i = idm_free_term(K.comfort_acc_max, r.speed, r.target_speed, P.lanes[lane].speed_limit, r.delta);
            int f_own, r_own;
            neighbours(P, F, V, lane, i, f_own, r_own);
            if constexpr (LINEAR) {
                acc = linear_acceleration(P, K, F, aligned, lsm->acc[0][i], lsm->acc[1][i], lsm->acc[2][i], i, f_own);
            } else {
                acc = free_i;  // behavior.py:115-120
                if (f_own >= 0) acc -= idm_gap_term(P, K, F, aligned, i, f_own);
            }
            if (lane != tgt0) {
                // change_lane_policy, ongoing change (behavior.py:229-244).  Only a controlled
                // vehicle v that is not on our target lane T and whose target is T when we act
                // can abort us: candidates = (target is T now) or (may switch to T this act).
                is_mid = true;
                uint32_t g[NW];
#pragma unroll
                for (int w = 0; w < NW; ++w) {
                    uint32_t may = F.tm[tgt0][w];
                    uint32_t adj = (tgt0 > 0 ? F.lane_is[tgt0 - 1][w] : 0u) |
                                   (tgt0 < P.lanes_count - 1 ? F.lane_is[tgt0 + 1][w] : 0u);
                    may |= F.fired[w] & adj;
                    uint32_t cand = may & sm.ctrl[w] & ~F.lane_is[tgt0][w];
                    if (w == (i >> 5)) cand &= ~(1u << (i & 31));
                    g[w] = 0;
                    while (cand) {
                        int b = __ffs(cand) - 1;
                        cand &= cand - 1;
                        int v = w * 32 + b;
                        double d = lane_distance(P, F, aligned, i, v);
                        double d_star = desired_gap(K, F, i, v);
                        if (0 < d && d < d_star) g[w] |= 1u << b;
                    }
                    sm.geo[i][w] = g[w];
                }
                atomicOr(&sm.mid[i >> 5], 1u << (i & 31));
            } else if (P.lane_change_delay < r.timer) {  // utils.do_every (utils.py:27-28)
                r.timer = 0.0;
                fired = true;
                // side_lanes (road/road.py:200-211): id-1 then id+1.  Each admissible candidate
                // becomes a work item; mobil() itself runs in phase A2 on a dense set of threads.
                sm.free_t[i] = free_i;
                sm.acc_own[i] = acc;
                sm.f_own[i] = (signed char)f_own;
                sm.r_own[i] = (signed char)r_own;
                if (!(fabs(r.speed) < 1)) {
                    for (int k = 0; k < 2; ++k) {
                        int cand = k == 0 ? lane - 1 : lane + 1;
                        if (cand < 0 || cand > P.lanes_count - 1) continue;
                        if (!lane_reachable(P.lanes[cand], r.x, r.y)) continue;
                        int slot_ = atomicAdd(&sm.n_items, 1);
                        sm.items[slot_] = (unsigned short)(i | (cand << 8) | (k << 15));
                    }
                }
            }
        }
        PHASE_MARK(7);  // phase A1
        env_sync_phase<TPE, 2>();
        PHASE_MARK(8);  // barrier after phase A1

        // ---- phase A2: mobil(lane_index) (behavior.py:265-324; route None => acceleration-gain
        // branch) for the queued (vehicle, candidate) items, one item per thread.
        if constexpr (LINEAR) {
            // the same with LinearVehicle.acceleration (behavior.py:417-465) and the item owner's parameters
            for (int t = i; (!DENSE || active) && t < sm.n_items; t += DENSE ? V : TPE) {
                const int it = sm.items[t];
                const int v = it & 0xff, cand = (it >> 8) & 0x7f, right = it >> 15;
                const double a0 = lsm->acc[0][v], a1 = lsm->acc[1][v], a2 = lsm->acc[2][v];
                int new_preceding, new_following;
                neighbours_cold(P, F, V, cand, v, new_preceding, new_following);
                double new_following_pred_a =
                    linear_acceleration(P, K, F, aligned, a0, a1, a2, new_following, v);
                if (new_following_pred_a < -P.lane_change_max_braking_imposed) continue;
                double self_pred_a = linear_acceleration(P, K, F, aligned, a0, a1, a2, v, new_preceding);
                double self_a = sm.acc_own[v];  // acceleration(self, old_preceding)
                double jerk = self_pred_a - self_a;
                if (P.politeness != 0.0) {
                    const int f_o = sm.f_own[v], r_o = sm.r_own[v];
                    double new_following_a =
                        linear_acceleration(P, K, F, aligned, a0, a1, a2, new_following, new_preceding);
                    double old_following_a = linear_acceleration(P, K, F, aligned, a0, a1, a2, r_o, v);
                    double old_following_pred_a = linear_acceleration(P, K, F, aligned, a0, a1, a2, r_o, f_o);
                    jerk = self_pred_a - self_a +
                           P.politeness * (new_following_pred_a - new_following_a + old_following_pred_a -
                                           old_following_a);
                }
                if (jerk < P.lane_change_min_acc_gain) continue;
                atomicOr(right ? &sm.ok_right[v >> 5] : &sm.ok_left[v >> 5], 1u << (v & 31));
            }
        } else
        for (int t = i; (!DENSE || active) && t < sm.n_items; t += DENSE ? V : TPE) {
            const int it = sm.items[t];
            const int v = it & 0xff, cand = (it >> 8) & 0x7f, right = it >> 15;
            const double delta_v = sm.delta[v];
            int new_preceding, new_following;
            neighbours_cold(P, F, V, cand, v, new_preceding, new_following);
            double new_following_pred_a = idm_acceleration_of(P, K, F, aligned, delta_v, new_following, v);
            if (new_following_pred_a < -P.lane_change_max_braking_imposed) continue;
            double self_pred_a = sm.free_t[v];
            if (new_preceding >= 0) self_pred_a -= idm_gap_term(P, K, F, aligned, v, new_preceding);
            double self_a = sm.acc_own[v];  // acceleration(self, old_preceding)
            double jerk = self_pred_a - self_a;
            if (P.politeness != 0.0) {
                const int f_o = sm.f_own[v], r_o = sm.r_own[v];
                double new_following_a =
                    idm_acceleration_of(P, K, F, aligned, delta_v, new_following, new_preceding);
                double old_following_a = idm_acceleration_of(P, K, F, aligned, delta_v, r_o, v);
                double old_following_pred_a = idm_acceleration_of(P, K, F, aligned, delta_v, r_o, f_o);
                jerk = self_pred_a - self_a +
                       P.politeness * (new_following_pred_a - new_following_a + old_following_pred_a -
                                       old_following_a);
            }
            if (jerk < P.lane_change_min_acc_gain) continue;
            atomicOr(right ? &sm.ok_right[v >> 5] : &sm.ok_left[v >> 5], 1u << (v & 31));
        }
        PHASE_MARK(13);  // phase A2
        env_sync_phase<TPE, 2>();
        PHASE_MARK(14);  // barrier after phase A2

        // ---- Road.act() phase B (steering + target-lane IDM with the final target), then
        // Road.step(dt): Vehicle.step (kinematics.py:130-177; IDMVehicle.step behavior.py:139-148).
        // The new state goes to the other frame, so no barrier is needed before staging it.
        if (active) {
            // both side lanes may pass mobil(); the later one (id+1) wins (behavior.py:252-263)
            int tgt = tgt0;
            if (fired) {
                if (test_bit(sm.ok_right, i))
                    tgt = lane + 1;
                else if (test_bit(sm.ok_left, i))
                    tgt = lane - 1;
            }
            if (is_mid) {
                // Ordered resolution of the Gauss-Seidel abort scan (behavior.py:229-244).  Vehicles
                // act in list order: vehicle j sees the NEW target of every earlier vehicle and the
                // OLD one of every later vehicle.  Only events on our target lane T matter (a
                // vehicle leaving T, or an aborting vehicle returning to its own lane, sits ON the
                // lane it now targets and is excluded by `lane_index != T`), so each mid-change
                // vehicle replays, redundantly and in registers, the decisions of the earlier
                // mid-change vehicles that share its target.
                const int T = tgt0, iw = i >> 5, ib = i & 31;
                uint32_t tmT[NW], lneT[NW], chgT[NW], ab[NW];
#pragma unroll
                for (int w = 0; w < NW; ++w) {
                    tmT[w] = F.tm[T][w];
                    lneT[w] = ~F.lane_is[T][w];
                    // vehicles whose MOBIL decision just switched their target to T
                    chgT[w] = (T > 0 ? sm.ok_right[w] & F.lane_is[T - 1][w] : 0u) |
                              (T < P.lanes_count - 1 ? sm.ok_left[w] & ~sm.ok_right[w] & F.lane_is[T + 1][w] : 0u);
                    ab[w] = 0;
                }
#pragma unroll
                for (int w = 0; w < NW; ++w) {
                    uint32_t m = sm.mid[w] & tmT[w];
                    if (w > iw) m = 0;
                    if (w == iw) m &= (2u << ib) - 1u;  // mids up to and including ourselves
                    while (m) {
                        int b = __ffs(m) - 1;
                        m &= m - 1;
                        int j = w * 32 + b;
                        uint32_t hit = 0;
#pragma unroll
                        for (int w2 = 0; w2 < NW; ++w2) {
                            uint32_t below = w2 < w ? ~0u : (w2 == w ? (1u << b) - 1u : 0u);
                            uint32_t cur = (tmT[w2] & ~ab[w2]) | (chgT[w2] & below);
                            hit |= sm.geo[j][w2] & lneT[w2] & cur;
                        }
                        if (hit) ab[w] |= 1u << b;  // behavior.py:241-243: target := current lane
                    }
                }
                if ((ab[iw] >> ib) & 1u) tgt = lane;
            }
            // IDMVehicle.act (behavior.py:109-112) and ControlledVehicle.act(None)
            // (controller.py:126-133, runs even when crashed) share the steering law
            double sin_beta = 0.0, cos_beta = 1.0;  // crashed: steering 0 (clip_actions :155-158)
            if constexpr (LINEAR) {
                // LinearVehicle.steering_control is an explicit (clipped) angle: Vehicle.step's arctan(tan / 2)
                if (idm_active) {
                    beta_of_angle(linear_steering(P.lanes[tgt], r.x, r.y, r.heading, r.speed, lsm->steer[0][i],
                                                  lsm->steer[1][i]),
                                  sin_beta, cos_beta);
                } else if (kind == HWY_KIND_MDP && !crashed) {
                    double xs = steering_sin_slip(P.lanes[tgt], r.x, r.y, r.heading, r.speed);
                    beta_of_controlled(xs, sin_beta, cos_beta);
                } else if (kind == HWY_KIND_VEHICLE && !crashed) {
                    beta_of_angle(act_steer, sin_beta, cos_beta);
                }
            } else
            if (idm_active || (kind == HWY_KIND_MDP && !crashed)) {
                double xs = steering_sin_slip(P.lanes[tgt], r.x, r.y, r.heading, r.speed);
                beta_of_controlled(xs, sin_beta, cos_beta);
            } else if (kind == HWY_KIND_VEHICLE && !crashed) {
                beta_of_angle(act_steer, sin_beta, cos_beta);
            }
            if (idm_active) {
                if (lane != tgt) {  // behavior.py:121-131
                    int f_t, r_t;
                    neighbours_cold(P, F, V, tgt, i, f_t, r_t);
                    double tacc;
                    if constexpr (LINEAR) {
                        tacc = linear_acceleration(P, K, F, aligned, lsm->acc[0][i], lsm->acc[1][i], lsm->acc[2][i], i,
                                                   f_t);
                    } else {
                        tacc = free_i;
                        if (f_t >= 0) tacc -= idm_gap_term(P, K, F, aligned, i, f_t);
                    }
                    acc = fmin(acc, tacc);
                }
                act_accel = clipd(acc, -P.acc_max, P.acc_max);
            } else if (kind == HWY_KIND_MDP) {
                act_accel = kKpA * (r.target_speed - r.speed);  // speed_control :189-198
            }
            r.meta = meta_set_target(r.meta, tgt);

            PHASE_MARK(9);  // phase B
            if (kind == HWY_KIND_IDM) r.timer += dt;
            if (crashed) {  // clip_actions :155-168
                act_steer = 0.0;
                act_accel = -1.0 * r.speed;
            }
            if (r.speed > kMaxSpeed)
                act_accel = fmin(act_accel, 1.0 * (kMaxSpeed - r.speed));
            else if (r.speed < kMinSpeed)
                act_accel = fmax(act_accel, 1.0 * (kMinSpeed - r.speed));
            // cos/sin(heading + beta) by angle addition from the staged cos/sin(heading)
            const double ch = F.c[i], sh = F.s[i];
            double cs = ch * cos_beta - sh * sin_beta, sn = sh * cos_beta + ch * sin_beta;
            double vx = r.speed * cs, vy = r.speed * sn;
            r.x += vx * dt;
            r.y += vy * dt;
            if (r.meta & HWY_META_HAS_IMPACT) {
                r.x += r.imp_x;
                r.y += r.imp_y;
                r.meta = (r.meta | HWY_META_CRASHED) & ~HWY_META_HAS_IMPACT;
            }
            r.heading += div_finite(r.speed * sin_beta, kVehLength / 2) * dt;
            r.speed += act_accel * dt;
            int nl = closest_lane(P, r.x, r.y, r.heading, congruent);  // on_state_update :170-177
            r.meta = meta_set_lane(r.meta, nl);
            if (kind == HWY_KIND_VEHICLE) r.meta = meta_set_target(r.meta, nl);  // schema: mirrors lane
        }
        PHASE_MARK(10);  // integrate
    }

    PHASE_MARK(11);
    // the final frame's road order goes back with the state, for frame 0 of the next launch
    if (active) r.meta = meta_set_order(r.meta, sm.f[p].perm[i]);
    if (substeps_only) {  // uniform over the grid
        if (active && env_ok) store_vehicle(S, slot, r);
        return;
    }
    // ---- epilogue: state back to HBM, observation, reward, termination
    const Frame<TPE>& F = sm.f[p];
    const size_t obs_off = (size_t)e * P.obs_vehicles_count * obs_columns(P);
    float* obs_env = obs + obs_off;
    // MULTI: one observation per controlled vehicle as observer under multi_obs (observation.py:588-604), else the
    // first one's; rows [n_envs][NA][K][columns]
    const int NA = MULTI && P.multi_obs ? P.n_agents : 1;
    if constexpr (MULTI) {
        for (int a = 0; a < NA; ++a) {
            const size_t off = ((size_t)e * NA + a) * P.obs_vehicles_count * obs_columns(P);
            kinematics_observe<TPE, DENSE>(P, F, sm.key, i, r.heading, env_ok ? obs + off : nullptr,
                                           (autoreset && final_obs) ? final_obs + off : nullptr,
                                           nth_controlled(msm->ego, a));
            env_sync<TPE>();  // the next observer's keys overwrite sm.key
        }
    } else
    kinematics_observe<TPE, DENSE>(P, F, sm.key, i, r.heading, env_ok ? obs_env : nullptr,
                       (autoreset && final_obs) ? final_obs + obs_off : nullptr);
    if (i == 0) {
        sm.done = 0;
        sm.sp_fallback = 0;
    }
    if (i == 0 && env_ok) {
        // envs/highway_env.py:100-151
        const int lane = meta_lane(r.meta);
        const HwyStraightLane& L = P.lanes[lane];
        int rl = kind == HWY_KIND_VEHICLE ? lane : meta_target(r.meta);
        double forward_speed = r.speed * F.c[0];
        double scaled_speed = lmap(forward_speed, P.reward_speed_lo, P.reward_speed_hi, 0.0, 1.0);
        double es, elat;
        lane_local(L, r.x, r.y, es, elat);
        bool on_road = lane_on(L, es, elat, 0.0);
        bool is_crashed = (r.meta & HWY_META_CRASHED) != 0;
        int nl1 = P.lanes_count - 1 > 1 ? P.lanes_count - 1 : 1;
        double rew = 0.0;
        rew = rew + P.collision_reward * (is_crashed ? 1.0 : 0.0);
        rew = rew + P.right_lane_reward * ((double)rl / (double)nl1);
        rew = rew + P.high_speed_reward * clipd(scaled_speed, 0.0, 1.0);
        rew = rew + 0.0 * (on_road ? 1.0 : 0.0);
        if (P.normalize_reward)
            rew = lmap(rew, P.collision_reward, P.high_speed_reward + P.right_lane_reward, 0.0, 1.0);
        rew *= on_road ? 1.0 : 0.0;
        double t = S.time[e] + 1.0 / P.policy_frequency;  // abstract.py:274
        S.time[e] = t;
        if constexpr (!MULTI) S.speed_index[e] = speed_index;
        reward[e] = rew;
        terminated[e] = (uint8_t)(is_crashed || (P.offroad_terminal && !on_road));
        truncated[e] = (uint8_t)(t >= P.duration);
        if (info_speed) info_speed[e] = r.speed;  // abstract.py:200-217 _info
        if (info_crashed) info_crashed[e] = (uint8_t)is_crashed;
        if (S.reward_terms) {  // _rewards (highway_env.py:118-137): info["rewards"]
            double* rt = S.reward_terms + (size_t)e * HWY_REWARD_TERMS;
            rt[0] = is_crashed ? 1.0 : 0.0;
            rt[1] = (double)rl / (double)nl1;
            rt[2] = clipd(scaled_speed, 0.0, 1.0);
            rt[3] = on_road ? 1.0 : 0.0;
            rt[4] = 0.0;
        }
        sm.done = autoreset && (is_crashed || (P.offroad_terminal && !on_road) || t >= P.duration);
    }
    if constexpr (MULTI)
        if (controlled && env_ok && agent < P.n_agents) S.speed_index[(size_t)e * P.n_agents + agent] = speed_index;
    if (autoreset) {
        // ---- SameStep autoreset fused into the step: envs that ended re-spawn from their own
        // numpy stream and return the reset observation (gymnasium AutoresetMode.SAME_STEP)
        env_sync<TPE>();
        const bool do_reset = env_ok && sm.done;
        const bool simple_geometry = aligned && P.lanes[0].start_x == 0.0 && P.lanes[0].dir_x == 1.0;
        spawn_fused<TPE, LINEAR, MULTI>(P, S, sm, e, i, active, do_reset, simple_geometry, r, speed_index, T);
        Frame<TPE>& G = sm.f[p ^ 1];
        if (do_reset) publish<TPE, false, DENSE>(P, G, i, active, r);
        // barrier + "does any env of this block re-spawn?": the second observation runs under a block-uniform
        // condition, so that all threads of the block meet the same barrier instructions (a per-env condition around
        // __syncthreads() is what compute-sanitizer's synccheck rejects, even though the arrival counts match)
        const bool any_reset = __syncthreads_or(do_reset) != 0;
        if (any_reset) {
            if constexpr (MULTI) {  // the respawned layout: controlled vehicle a at spawn_ego_slot(a)
                for (int a = 0; a < NA; ++a) {
                    const size_t off = ((size_t)e * NA + a) * P.obs_vehicles_count * obs_columns(P);
                    kinematics_observe<TPE, DENSE>(P, G, sm.key, i, r.heading, do_reset ? obs + off : nullptr,
                                                   nullptr, spawn_ego_slot(V, P.n_agents, a));
                    env_sync<TPE>();
                }
                if (do_reset && i == 0) S.time[e] = 0.0;
                bool ego;
                const int ag = spawn_bin(V, P.n_agents, i, ego);
                if (do_reset && active && ego) S.speed_index[(size_t)e * P.n_agents + ag] = speed_index;
            } else {
            kinematics_observe<TPE, DENSE>(P, G, sm.key, i, r.heading, do_reset ? obs_env : nullptr);
            if (do_reset && i == 0) {
                S.time[e] = 0.0;
                S.speed_index[e] = speed_index;
            }
            }
        }
    }
    if (active && env_ok) store_vehicle(S, slot, r);
    if (autoreset && active && env_ok && sm.done) S.delta[slot] = r.delta;
    PHASE_MARK(12);  // epilogue
