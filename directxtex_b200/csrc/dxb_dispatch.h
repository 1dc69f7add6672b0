// dxb_dispatch.h — run-time values to template arguments.  A launcher states the instantiations it compiles once, as the
// template arguments of one of these calls, and launches its kernel inside a generic lambda that reads them back with
// decltype(arg)::value.
#pragma once
#include <stdint.h>
#include <type_traits>

template <uint32_t V> using dxb_u32 = std::integral_constant<uint32_t, V>;

// fn(dxb_u32<F>{}) for the F of the list equal to f; false when none is
template <uint32_t... Fs, typename Fn>
bool dxb_on_value(uint32_t f, Fn&& fn)
{
    return ((f == Fs ? (fn(dxb_u32<Fs>{}), true) : false) || ...);
}

// the list is A0, B0, A1, B1, ...: fn(dxb_u32<A>{}, dxb_u32<B>{}) for the pair equal to (a, b); false when none is
template <uint32_t A, uint32_t B, uint32_t... Rest, typename Fn>
bool dxb_on_pair(uint32_t a, uint32_t b, Fn&& fn)
{
    if (a == A && b == B) { fn(dxb_u32<A>{}, dxb_u32<B>{}); return true; }
    if constexpr (sizeof...(Rest) > 0) return dxb_on_pair<Rest...>(a, b, fn);
    else return false;
}

// fn(std::true_type{}) or fn(std::false_type{}); returns what fn returns
template <typename Fn>
auto dxb_on_bool(bool b, Fn&& fn)
{
    if (b) return fn(std::true_type{});
    return fn(std::false_type{});
}
