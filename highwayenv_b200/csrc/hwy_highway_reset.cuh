// hwy_highway_reset.cuh — the body of the highway reset kernels, included by highway_reset_kernel (LINEAR = false)
// and highway_linear_reset_kernel (LINEAR = true) in hwy_highway.cu.  In scope: LINEAR, the kernel parameters and
// `const HwyLinearTraffic* T`.
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= S.n_envs || !env_selected(mask_a, mask_b, e)) return;
    Pcg64 g = load_rng(S.rng, (size_t)S.n_envs, e);

    double x_max = 0.0;  // running max of the longitudinal coordinates of spawned vehicles
    bool aligned = true;  // all lanes share origin-x and direction => s is lane independent
    for (int l = 1; l < P.lanes_count; ++l)
        aligned = aligned && P.lanes[l].start_x == P.lanes[0].start_x &&
                        P.lanes[l].dir_x == P.lanes[0].dir_x && P.lanes[l].dir_y == 0.0 &&
                        P.lanes[0].dir_y == 0.0;
    double2* pos = reinterpret_cast<double2*>(S.pos);
    double2* hs = reinterpret_cast<double2*>(S.hs);
    double2* tt = reinterpret_cast<double2*>(S.tt);
    double2* imp = reinterpret_cast<double2*>(S.imp);
    const size_t base = (size_t)e * S.vp;
    int ego_speed_index = -1;
    for (int v = 0; v < P.n_vehicles; ++v) {
        const bool is_ego = v == 0;
        // choice(list(graph.keys())) / choice(list(graph[_from].keys())): single element => no draw
        int id = (is_ego && P.initial_lane_id >= 0) ? P.initial_lane_id : g.choice(P.lanes_count);
        const HwyStraightLane& L = P.lanes[id];
        double speed = is_ego ? P.ego_speed : g.uniform(0.7 * L.speed_limit, 0.8 * L.speed_limit);
        double spacing = is_ego ? P.ego_spacing : 1 / P.vehicles_density;
        double default_spacing = 12 + 1.0 * speed;
        double offset = spacing * default_spacing * P.spawn_exp;
        double x0;
        if (v > 0) {
            if (aligned) {
                x0 = x_max;
            } else {  // np.max over lane.local_coordinates(v.position)[0] on the chosen lane
                x0 = lane_s(L, pos[base].x, pos[base].y);
                for (int j = 1; j < v; ++j) x0 = fmax(x0, lane_s(L, pos[base + j].x, pos[base + j].y));
            }
        } else {
            x0 = 3 * offset;
        }
        x0 += offset * g.uniform(0.9, 1.1);
        // lane.position(x0, 0), lane.heading_at(x0)  (road/lane.py:192-200)
        double px = (L.start_x + x0 * L.dir_x) + 0.0 * L.lat_x;
        double py = (L.start_y + x0 * L.dir_y) + 0.0 * L.lat_y;
        double heading = L.heading;
        double s_here = lane_s(L, px, py);
        x_max = v == 0 ? s_here : fmax(x_max, s_here);
        int lane = closest_lane(P, px, py, heading);  // RoadObject.__init__ objects.py:46-50
        double target_speed = speed;                   // `target_speed or self.speed`
        double timer = 0.0, delta = 4.0;
        double lin[HWY_LINEAR_PARAMS] = {0.0, 0.0, 0.0, 0.0, 0.0};
        int kind, cc;
        if (is_ego) {
            cc = 1;
            if (P.action_type == 0) {
                kind = HWY_KIND_MDP;
                ego_speed_index = speed_to_index(P, target_speed);
                target_speed = P.target_speeds[ego_speed_index];
            } else {
                kind = HWY_KIND_VEHICLE;
            }
        } else {
            kind = HWY_KIND_IDM;
            cc = P.others_check_collisions;
            timer = py_mod_pos((px + py) * kPi, P.lane_change_delay);  // behavior.py:64
            if constexpr (LINEAR) draw_linear_params(g, *T, lin);
            delta = g.uniform(P.delta_lo, P.delta_hi);                 // behavior.py:66-69
        }
        if constexpr (LINEAR)
            for (int k = 0; k < HWY_LINEAR_PARAMS; ++k) T->params[(base + v) * HWY_LINEAR_PARAMS + k] = lin[k];
        pos[base + v] = make_double2(px, py);
        hs[base + v] = make_double2(heading, speed);
        tt[base + v] = make_double2(target_speed, timer);
        imp[base + v] = make_double2(0.0, 0.0);
        S.delta[base + v] = delta;
        S.meta[base + v] = (lane << HWY_META_LANE_SHIFT) | (lane << HWY_META_TARGET_SHIFT) |
                           (cc ? HWY_META_CHECK_COLLISIONS : 0) | (kind << HWY_META_KIND_SHIFT) |
                           HWY_META_PRESENT;
    }
    S.speed_index[e] = ego_speed_index;
    S.time[e] = 0.0;
    store_rng_all(S.rng, (size_t)S.n_envs, e, g);
